// Fused epilogue of the 2D-CTC head (decoders/ctc_decoder2d.py:37-45, SURVEY.md section 8 row N2):
//
//     mask     = softmax_H(mask_logits)          [N,1,H,W]      (nn.Softmax(dim=2) at the end of pred_mask, :21)
//     classify = softmax_C(classify_logits)      [N,C,H,W]      (:41)
//     pred     = log(max(mask * classify, tiny)) [N,C,H,W]      (:43-44)
//     log_probs = pred.permute(3,2,0,1).contiguous()   -> [W,H,N,C] = the (T,H,N,C) operand of ctc_loss_2d   (:45)
//
// The reference runs this as two softmax kernels, a product, a max, a log and a permuting copy: 6 passes over
// N*C*H*W floats.  Here: ONE pass forward (read the NCHW logits once, write (T,H,N,C) once) and one pass backward
// (+ a tiny per-column fix-up for the mask branch).  The backward can take the 2D-CTC training factor `gfac`
// directly (grad[t,h,n,c] = exp(log_probs) * gfac[t,n,c] * grad_out[n], include/megreader_b200.h) so that the loss
// gradient w.r.t. log_probs never exists in HBM.
//
// Tiling: a block owns (NT samples) x (one height) x (32 columns); the NCHW side is read / written as 128-byte rows
// along W, the (T,H,N,C) side as NT*C contiguous floats per column, with a padded shared-memory tile in between.
// HBM-bound: algorithmic bytes per sample = 2*C*H*W*4 (+ mask) forward, 3*C*H*W*4 backward with explicit grad,
// 2*C*H*W*4 + T*C*4 with gfac.
#include "common.cuh"
#include <math.h>
#include <stdlib.h>
#include <algorithm>

namespace {
using namespace mr;

constexpr int kTW = 32;          // columns per block (tile row stride kTW + 1 = 33 floats)
constexpr int kThreads = 256;

struct HeadGeo { int N, C, H, W, NT; };

__device__ __forceinline__ float ex2f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2f(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;
// base + i * stride_bytes with a 32 x 32 -> 64-bit multiply-add: ONE IMAD.WIDE.U32 per address (the plain pointer + int form
// costs 5-7 integer instructions per access, which dominated the instruction count of these kernels)
__device__ __forceinline__ const float *at(const float *base, unsigned i, unsigned stride_bytes) {
    return reinterpret_cast<const float *>(reinterpret_cast<const char *>(base) + (uint64_t)i * stride_bytes);
}
__device__ __forceinline__ float *at(float *base, unsigned i, unsigned stride_bytes) {
    return reinterpret_cast<float *>(reinterpret_cast<char *>(base) + (uint64_t)i * stride_bytes);
}

// mask tile mt[nl][k][w] <- mask_logits[n0+nl, 0, k, w0+w]: all heights of the block's samples / columns (the softmax over
// H needs every height); loaded with the logits tile so that no thread waits on a chain of dependent global loads.
__device__ __forceinline__ void load_mask_tile(const HeadGeo &g, const float *__restrict__ m, int n0, int w0, float *mt) {
    const int w = threadIdx.x & 31, r0 = threadIdx.x >> 5;
    const int rows = g.NT * g.H;
    constexpr int RS = kThreads / 32, B = 8;
    for (int rb = r0; rb < rows; rb += RS * B) {
        float v[B];
#pragma unroll
        for (int j = 0; j < B; ++j) {
            const int r = rb + j * RS;
            const int nl = r / g.H, k = r - nl * g.H;
            const int n = n0 + nl;
            v[j] = 0.f;
            if (r < rows && n < g.N && w0 + w < g.W) v[j] = __ldg(m + ((int64_t)n * g.H + k) * g.W + w0 + w);
        }
#pragma unroll
        for (int j = 0; j < B; ++j) {
            const int r = rb + j * RS;
            if (r < rows) mt[r * (kTW + 1) + w] = v[j];
        }
    }
}
// log-probability (natural log) of height h under softmax_H of the mask column held in mt
__device__ __forceinline__ float mask_logsoftmax(const float *mt, int nl, int h, int w, int H) {
    const float *col = mt + (nl * H) * (kTW + 1) + w;
    float mx = -INFINITY;
    for (int k = 0; k < H; ++k) mx = fmaxf(mx, col[k * (kTW + 1)]);
    float s = 0.f;
    for (int k = 0; k < H; ++k) s += ex2f((col[k * (kTW + 1)] - mx) * kLog2e);
    return col[h * (kTW + 1)] - mx - lg2f(s) * kLn2;
}

// max and sum of 2^(v*log2e - max) over one tile column (stride kTW+1), four independent chains
__device__ __forceinline__ void column_max_sum(const float *col, int C, float &mx, float &s) {
    constexpr int ST = 33;
    float m0 = -INFINITY, m1 = -INFINITY, m2 = -INFINITY, m3 = -INFINITY;
    int c = 0;
    for (; c + 4 <= C; c += 4) {
        m0 = fmaxf(m0, col[c * ST]); m1 = fmaxf(m1, col[(c + 1) * ST]);
        m2 = fmaxf(m2, col[(c + 2) * ST]); m3 = fmaxf(m3, col[(c + 3) * ST]);
    }
    for (; c < C; ++c) m0 = fmaxf(m0, col[c * ST]);
    mx = fmaxf(fmaxf(m0, m1), fmaxf(m2, m3));
    const float off = mx * kLog2e;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    c = 0;
    for (; c + 4 <= C; c += 4) {
        s0 += ex2f(fmaf(col[c * ST], kLog2e, -off)); s1 += ex2f(fmaf(col[(c + 1) * ST], kLog2e, -off));
        s2 += ex2f(fmaf(col[(c + 2) * ST], kLog2e, -off)); s3 += ex2f(fmaf(col[(c + 3) * ST], kLog2e, -off));
    }
    for (; c < C; ++c) s0 += ex2f(fmaf(col[c * ST], kLog2e, -off));
    s = (s0 + s1) + (s2 + s3);
}

// tile[nl][c][w] <-> z[n0+nl, c, h, w0+w]  (rows of 32 floats along W)
__device__ __forceinline__ void load_nchw_tile(const HeadGeo &g, const float *__restrict__ z, int n0, int h, int w0,
                                               float *tile) {
    // batches of 8 independent loads per thread before the first shared-memory store: a load -> store loop body makes
    // every iteration wait for its own load (38 serialised memory latencies per block)
    const int w = threadIdx.x & 31, r0 = threadIdx.x >> 5;
    const int rows = g.NT * g.C;
    constexpr int RS = kThreads / 32, B = 20;           // 8 samples x 38 classes = 304 rows = 2 batches per thread
    for (int rb = r0; rb < rows; rb += RS * B) {
        float v[B];
#pragma unroll
        for (int j = 0; j < B; ++j) {
            const int r = rb + j * RS;
            const int nl = r / g.C, c = r - nl * g.C;
            const int n = n0 + nl;
            v[j] = 0.f;
            if (r < rows && n < g.N && w0 + w < g.W) v[j] = __ldg(z + (((int64_t)n * g.C + c) * g.H + h) * g.W + w0 + w);
        }
#pragma unroll
        for (int j = 0; j < B; ++j) {
            const int r = rb + j * RS;
            if (r < rows) tile[r * (kTW + 1) + w] = v[j];
        }
    }
}

// tile[e][w] <- src_w[e] for the 32 columns of the block, src_w = base + w * col_stride (NT*C contiguous floats each)
__device__ __forceinline__ void load_thnc_tile(const float *__restrict__ base, int64_t col_stride, int ncols, int per_col,
                                               int nvalid, float *tile) {
    constexpr int B = 16;
    for (int e0 = threadIdx.x; e0 < per_col; e0 += kThreads) {
        for (int wb = 0; wb < ncols; wb += B) {
            float v[B];
#pragma unroll
            for (int j = 0; j < B; ++j) {
                v[j] = 0.f;
                if (wb + j < ncols && e0 < nvalid) v[j] = __ldg(base + (int64_t)(wb + j) * col_stride + e0);
            }
#pragma unroll
            for (int j = 0; j < B; ++j)
                if (wb + j < kTW) tile[e0 * (kTW + 1) + wb + j] = v[j];
        }
    }
}

__device__ __forceinline__ void store_nchw_tile(const HeadGeo &g, float *__restrict__ z, int n0, int h, int w0,
                                                const float *tile) {
    const int w = threadIdx.x & 31, r0 = threadIdx.x >> 5;
    const int rows = g.NT * g.C;
    for (int r = r0; r < rows; r += kThreads / 32) {
        const int nl = r / g.C, c = r - nl * g.C;
        const int n = n0 + nl;
        if (n < g.N && w0 + w < g.W) z[(((int64_t)n * g.C + c) * g.H + h) * g.W + w0 + w] = tile[r * (kTW + 1) + w];
    }
}

// forward: logits -> log_probs (T=W, H, N, C)
__global__ void __launch_bounds__(kThreads)
ctc2d_head_fwd_kernel(HeadGeo g, const float *__restrict__ mask_logits, const float *__restrict__ cls_logits,
                      float log_tiny, float *__restrict__ lp) {
    extern __shared__ float tile[];                      // [NT*C][33] logits, then [NT*H][33] mask logits
    float *mt = tile + g.NT * g.C * (kTW + 1);
    const int w0 = blockIdx.x * kTW, h = blockIdx.y, n0 = blockIdx.z * g.NT;
    load_nchw_tile(g, cls_logits, n0, h, w0, tile);
    load_mask_tile(g, mask_logits, n0, w0, mt);
    __syncthreads();
    // one thread per (sample, column): class log-softmax + mask log-softmax, clamp at log(tiny)
    for (int item = threadIdx.x; item < g.NT * kTW; item += kThreads) {
        const int nl = item >> 5, w = item & 31;
        const int n = n0 + nl;
        if (n >= g.N || w0 + w >= g.W) continue;
        float *col = tile + (nl * g.C) * (kTW + 1) + w;
        float mx, sum;
        column_max_sum(col, g.C, mx, sum);
        // log(mask * classify) = z - max - ln(sum) + log mask ; one exponential per element in total
        const float shift = mask_logsoftmax(mt, nl, h, w, g.H) - mx - lg2f(sum) * kLn2;
#pragma unroll 4
        for (int c = 0; c < g.C; ++c) col[c * (kTW + 1)] = fmaxf(col[c * (kTW + 1)] + shift, log_tiny);
    }
    __syncthreads();
    // (T,H,N,C): for each column the NT*C values of this block are contiguous
    const int per_col = g.NT * g.C;
    const int nvalid = min(g.NT, g.N - n0) * g.C;
    for (int w = 0; w < kTW && w0 + w < g.W; ++w) {
        float *dst = lp + (((int64_t)(w0 + w) * g.H + h) * g.N + n0) * g.C;
        for (int e = threadIdx.x; e < per_col; e += kThreads)
            if (e < nvalid) dst[e] = tile[e * (kTW + 1) + w];
    }
}

// backward: d(log_probs) [or gfac/grad_out] -> d(classify logits) [N,C,H,W], and G[n,h,w] = sum_c g  (mask branch)
template <bool FACTORED>
__global__ void __launch_bounds__(kThreads)
ctc2d_head_bwd_kernel(HeadGeo g, const float *__restrict__ mask_logits, const float *__restrict__ cls_logits,
                      const float *__restrict__ dlp, const float *__restrict__ gfac, const float *__restrict__ go,
                      int64_t go_stride, float tiny, float *__restrict__ dcls, float *__restrict__ gsum) {
    extern __shared__ float smem[];
    const int per_col = g.NT * g.C;
    float *zt = smem;                                    // [NT*C][33] logits -> d logits
    float *gt = smem + per_col * (kTW + 1);              // [NT*C][33] upstream gradient (or factor)
    float *mt = gt + per_col * (kTW + 1);                // [NT*H][33] mask logits
    const int w0 = blockIdx.x * kTW, h = blockIdx.y, n0 = blockIdx.z * g.NT;
    load_nchw_tile(g, cls_logits, n0, h, w0, zt);
    load_mask_tile(g, mask_logits, n0, w0, mt);
    const int nvalid = min(g.NT, g.N - n0) * g.C;
    // explicit gradient is [T,H,N,C]; the factor is [T,N,C] (shared by all heights)
    if (FACTORED) load_thnc_tile(gfac + ((int64_t)w0 * g.N + n0) * g.C, (int64_t)g.N * g.C, min(kTW, g.W - w0), per_col, nvalid, gt);
    else load_thnc_tile(dlp + (((int64_t)w0 * g.H + h) * g.N + n0) * g.C, (int64_t)g.H * g.N * g.C, min(kTW, g.W - w0), per_col, nvalid, gt);
    __syncthreads();
    for (int item = threadIdx.x; item < g.NT * kTW; item += kThreads) {
        const int nl = item >> 5, w = item & 31;
        const int n = n0 + nl;
        if (n >= g.N || w0 + w >= g.W) continue;
        float *zc = zt + (nl * g.C) * (kTW + 1) + w;
        float *gc = gt + (nl * g.C) * (kTW + 1) + w;
        float mx, sum;
        column_max_sum(zc, g.C, mx, sum);
        const float inv = 1.f / sum, off = mx * kLog2e;
        const float maskp = ex2f(mask_logsoftmax(mt, nl, h, w, g.H) * kLog2e);
        const float gout = FACTORED ? __ldg(go + (int64_t)n * go_stride) : 1.f;
        // probability domain: p = classify prob, q = mask * p (what the reference clamps at tiny); max(q, tiny) passes no
        // gradient where q <= tiny.  With the CTC factor the upstream gradient is exp(log_probs) * gfac * go = q * gfac * go.
        float t0 = 0.f, t1 = 0.f;
        int c = 0;
        for (; c + 2 <= g.C; c += 2) {
            const float p0 = ex2f(fmaf(zc[c * (kTW + 1)], kLog2e, -off)) * inv;
            const float p1 = ex2f(fmaf(zc[(c + 1) * (kTW + 1)], kLog2e, -off)) * inv;
            const float q0 = p0 * maskp, q1 = p1 * maskp;
            const float u0 = gc[c * (kTW + 1)], u1 = gc[(c + 1) * (kTW + 1)];
            const float g0 = q0 > tiny ? (FACTORED ? q0 * u0 * gout : u0) : 0.f;
            const float g1 = q1 > tiny ? (FACTORED ? q1 * u1 * gout : u1) : 0.f;
            t0 += g0; t1 += g1;
            zc[c * (kTW + 1)] = p0; zc[(c + 1) * (kTW + 1)] = p1;
            gc[c * (kTW + 1)] = g0; gc[(c + 1) * (kTW + 1)] = g1;
        }
        for (; c < g.C; ++c) {
            const float p0 = ex2f(fmaf(zc[c * (kTW + 1)], kLog2e, -off)) * inv;
            const float q0 = p0 * maskp;
            const float u0 = gc[c * (kTW + 1)];
            const float g0 = q0 > tiny ? (FACTORED ? q0 * u0 * gout : u0) : 0.f;
            t0 += g0;
            zc[c * (kTW + 1)] = p0;
            gc[c * (kTW + 1)] = g0;
        }
        const float tot = t0 + t1;
#pragma unroll 4
        for (int k = 0; k < g.C; ++k) zc[k * (kTW + 1)] = gc[k * (kTW + 1)] - zc[k * (kTW + 1)] * tot;
        gsum[((int64_t)n * g.H + h) * g.W + w0 + w] = tot;
    }
    __syncthreads();
    store_nchw_tile(g, dcls, n0, h, w0, zt);
}

// mask branch: dm[n,h,w] = G[n,h,w] - softmax_H(m)[n,h,w] * sum_h' G[n,h',w]   (in place on G)
__global__ void ctc2d_head_mask_bwd_kernel(int N, int H, int W, const float *__restrict__ mask_logits, float *__restrict__ gm) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * W) return;
    const int n = (int)(i / W), w = (int)(i - (int64_t)n * W);
    const float *m = mask_logits + (int64_t)n * H * W + w;
    float *gp = gm + (int64_t)n * H * W + w;
    float mx = -INFINITY, tot = 0.f;
    for (int k = 0; k < H; ++k) { mx = fmaxf(mx, m[(int64_t)k * W]); tot += gp[(int64_t)k * W]; }
    float s = 0.f;
    for (int k = 0; k < H; ++k) s += ex2f((m[(int64_t)k * W] - mx) * kLog2e);
    const float inv = 1.f / s;
    for (int k = 0; k < H; ++k) gp[(int64_t)k * W] -= ex2f((m[(int64_t)k * W] - mx) * kLog2e) * inv * tot;
}

// =====================================================================================================
// Round-2 kernels: one WARP per slab (sample n, height h, 32 columns), lane = column.
//
// The block-tile kernels above run three barrier-separated phases per block and ~1000 instructions per thread around
// 4-byte accesses, far from the HBM roofline.
// Here a lane keeps ITS column's C class logits in registers: every global read of the NCHW side is a coalesced 128-byte
// row straight into registers (C + 2H independent loads in flight per lane, no staging), the softmax over C and the
// log-softmax of the mask column are register arithmetic, and only the (T,H,N,C) side -- whose contiguous direction is
// the class -- goes through a per-warp shared-memory transpose (odd pitch: conflict-free both ways).  No block barrier,
// no phases: the SM overlaps the loads of some warps with the arithmetic / stores of others.  CR = register rows (C <= CR);
// larger alphabets use the block-tile kernels above, and beyond their shared-memory tile the class-tiled kernels below.
// =====================================================================================================

__device__ __forceinline__ float mask_logsoftmax_col(const float *__restrict__ mcol, int H, int W, int h, bool valid) {
    // mcol = mask_logits + n*H*W + w ; two passes over the H rows (L1/L2 hits the second time): no register array
    if (!valid) return 0.f;
    float mx = -INFINITY;
    const float *p = mcol;
    for (int k = 0; k < H; ++k, p += W) mx = fmaxf(mx, __ldg(p));
    const float off = mx * kLog2e;
    float s = 0.f, mine = 0.f;
    p = mcol;
    for (int k = 0; k < H; ++k, p += W) {
        const float v = __ldg(p);
        s += ex2f(fmaf(v, kLog2e, -off));
        if (k == h) mine = v;
    }
    return mine - mx - lg2f(s) * kLn2;
}

// CX > 0: the alphabet size is exactly CX (compile time: every class predicate and address folds); CX = 0: runtime C <= CR.
template <int CR, int kWarpsPerBlock, int CX>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, CR <= 40 ? 3 : 2)
ctc2d_head_fwd_warp_kernel(HeadGeo g, const float *__restrict__ mask_logits, const float *__restrict__ cls_logits,
                           float log_tiny, float *__restrict__ lp) {
    constexpr int PITCH = CR + 1;                         // odd: lanes over columns write, lanes over classes read
    __shared__ float sm_all[kWarpsPerBlock][32 * PITCH];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float *sm = sm_all[warp];
    const int C = CX > 0 ? CX : g.C;
    const int wtiles = (g.W + 31) >> 5;
    const int64_t nslabs = (int64_t)g.N * g.H * wtiles;
    const int64_t HW = (int64_t)g.H * g.W;
    const unsigned HWB = (unsigned)(g.H * g.W) * 4u;       // byte strides; the host checks that they fit in 32 bits
    for (int64_t slab = (int64_t)blockIdx.x * kWarpsPerBlock + warp; slab < nslabs; slab += (int64_t)gridDim.x * kWarpsPerBlock) {
        // slab order: sample fastest -- the warps of a block (and neighbouring blocks) write the (T,H,N,C) rows of consecutive
        // samples at the same time, so the 152-byte per-sample pieces of a row merge into full sectors in L2
        const int n = (int)(slab % g.N);
        const int64_t hw = slab / g.N;
        const int wt = (int)(hw % wtiles);
        const int h = (int)(hw / wtiles);
        const int w0 = wt << 5, w = w0 + lane;
        const bool valid = w < g.W;
        const float *zp = cls_logits + ((int64_t)n * C * g.H + h) * g.W + w;      // + c * H * W
        float zr[CR];
#pragma unroll
        for (int c = 0; c < CR; ++c) zr[c] = (valid && c < C) ? __ldg(at(zp, c, HWB)) : -INFINITY;
        const float mlog = mask_logsoftmax_col(mask_logits + (int64_t)n * HW + w, g.H, g.W, h, valid);
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < CR; ++c) mx = fmaxf(mx, zr[c]);
        const float off = mx * kLog2e;
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int c = 0; c < CR; c += 2) {
            s0 += ex2f(fmaf(zr[c], kLog2e, -off));
            if (c + 1 < CR) s1 += ex2f(fmaf(zr[c + 1], kLog2e, -off));
        }
        // log(mask * classify) = z - max - ln(sum) + log mask ; one exponential per element in total
        const float shift = mlog - mx - lg2f(s0 + s1) * kLn2;
#pragma unroll
        for (int c = 0; c < CR; ++c)
            if (c < C) sm[lane * PITCH + c] = fmaxf(zr[c] + shift, log_tiny);
        __syncwarp();
        // (T,H,N,C): column w0+wl of this slab = C contiguous floats at (((w0+wl)*H + h)*N + n)*C
        const int ncol = min(32, g.W - w0);
        float *dst = lp + (((int64_t)w0 * g.H + h) * g.N + n) * C + lane;
        const unsigned cstepB = (unsigned)(g.H * g.N * C) * 4u;
        const bool c0ok = lane < C, c1ok = lane + 32 < C;              // C <= CR <= 64: two class passes
        const float *src = sm + lane;
#pragma unroll 8
        for (int wl = 0; wl < ncol; ++wl) {
            float *d = at(dst, wl, cstepB);
            if (c0ok) d[0] = src[wl * PITCH];
            if (c1ok) d[32] = src[wl * PITCH + 32];
        }
        __syncwarp();
    }
}

template <int CR, bool FACTORED, int kWarpsPerBlock, int CX>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, 2)     // 3 blocks / SM (80 registers) spills ~230 bytes per thread: slower
ctc2d_head_bwd_warp_kernel(HeadGeo g, const float *__restrict__ mask_logits, const float *__restrict__ cls_logits,
                           const float *__restrict__ dlp, const float *__restrict__ gfac, const float *__restrict__ go,
                           int64_t go_stride, float tiny, float *__restrict__ dcls, float *__restrict__ gsum) {
    constexpr int PITCH = CR + 1;
    __shared__ float sm_all[kWarpsPerBlock][32 * PITCH];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float *sm = sm_all[warp];
    const int C = CX > 0 ? CX : g.C;
    const int wtiles = (g.W + 31) >> 5;
    // explicit gradient: one slab = (sample, height, 32 columns).  CTC factor: the [T,N,C] tile is shared by all heights, so one
    // slab = (sample, 32 columns) and the heights are an inner loop over the staged tile (one eighth of the tile traffic).
    const int64_t nslabs = (int64_t)g.N * (FACTORED ? 1 : g.H) * wtiles;
    const int64_t HW = (int64_t)g.H * g.W;
    const unsigned HWB = (unsigned)(g.H * g.W) * 4u;       // byte strides; the host checks that they fit in 32 bits
    for (int64_t slab = (int64_t)blockIdx.x * kWarpsPerBlock + warp; slab < nslabs; slab += (int64_t)gridDim.x * kWarpsPerBlock) {
        const int n = (int)(slab % g.N);
        const int64_t hw = slab / g.N;
        const int wt = (int)(hw % wtiles);
        const int h_first = FACTORED ? 0 : (int)(hw / wtiles);
        const int h_end = FACTORED ? g.H : h_first + 1;
        const int w0 = wt << 5, w = w0 + lane;
        const bool valid = w < g.W;
        // upstream gradient (explicit [T,H,N,C]) or CTC factor ([T,N,C]): rows of C contiguous floats per column -> lanes over
        // classes load (16 columns = 32 loads in flight), lanes over columns read back
        {
            const int ncol = min(32, g.W - w0);
            const float *src = (FACTORED ? gfac + ((int64_t)w0 * g.N + n) * C : dlp + (((int64_t)w0 * g.H + h_first) * g.N + n) * C) + lane;
            const unsigned cstepB = (unsigned)(FACTORED ? g.N * C : g.H * g.N * C) * 4u;
            const bool c0ok = lane < C, c1ok = lane + 32 < C;
            float *d = sm + lane;
#pragma unroll 1
            for (int wl0 = 0; wl0 < 32; wl0 += 16, d += 16 * PITCH) {
                float a[16], b[16];
                const float *q = at(src, wl0, cstepB);
#pragma unroll
                for (int u = 0; u < 16; ++u) {
                    const bool in = wl0 + u < ncol;
                    a[u] = (in && c0ok) ? __ldg(at(q, u, cstepB)) : 0.f;
                    b[u] = (in && c1ok) ? __ldg(at(q, u, cstepB) + 32) : 0.f;
                }
#pragma unroll
                for (int u = 0; u < 16; ++u) {
                    d[u * PITCH] = a[u];
                    if (32 + lane < CR) d[u * PITCH + 32] = b[u];
                }
            }
        }
        __syncwarp();
        const float gout = (FACTORED && valid) ? __ldg(go + (int64_t)n * go_stride) : 1.f;
#pragma unroll 1
        for (int h = h_first; h < h_end; ++h) {
            const float *zp = cls_logits + ((int64_t)n * C * g.H + h) * g.W + w;
            float zr[CR];
#pragma unroll
            for (int c = 0; c < CR; ++c) zr[c] = (valid && c < C) ? __ldg(at(zp, c, HWB)) : -INFINITY;
            const float maskp = ex2f(mask_logsoftmax_col(mask_logits + (int64_t)n * HW + w, g.H, g.W, h, valid) * kLog2e);
            float mx = -INFINITY;
#pragma unroll
            for (int c = 0; c < CR; ++c) mx = fmaxf(mx, zr[c]);
            const float off = mx * kLog2e;
            float s0 = 0.f, s1 = 0.f;
#pragma unroll
            for (int c = 0; c < CR; c += 2) {
                zr[c] = ex2f(fmaf(zr[c], kLog2e, -off));          // zr becomes the un-normalised class probability
                s0 += zr[c];
                if (c + 1 < CR) { zr[c + 1] = ex2f(fmaf(zr[c + 1], kLog2e, -off)); s1 += zr[c + 1]; }
            }
            const float inv = 1.f / (s0 + s1);
            // probability domain: p = classify prob, q = mask * p (what the reference clamps at tiny); max(q, tiny) passes no
            // gradient where q <= tiny.  With the CTC factor the upstream gradient is exp(log_probs) * gfac * go = q * gfac * go.
            float t0 = 0.f, t1 = 0.f;
            float gr[CR];
#pragma unroll
            for (int c = 0; c < CR; ++c) {
                zr[c] *= inv;
                const float q = zr[c] * maskp;
                const float u = sm[lane * PITCH + c];
                gr[c] = (c < C && q > tiny) ? (FACTORED ? q * u * gout : u) : 0.f;
                if (c & 1) t1 += gr[c]; else t0 += gr[c];
            }
            const float tot = t0 + t1;
            if (valid) {
                float *op = dcls + ((int64_t)n * C * g.H + h) * g.W + w;
#pragma unroll
                for (int c = 0; c < CR; ++c)
                    if (c < C) *at(op, c, HWB) = gr[c] - zr[c] * tot;
                gsum[((int64_t)n * g.H + h) * g.W + w] = tot;
            }
        }
        __syncwarp();
    }
}

// =====================================================================================================
// Any alphabet (ChineseCharset, concern/charsets.py:65-78: ~5 k classes) and any H, W: class-TILED kernels.  A block owns one
// (sample, height, 32-column tile); warp k streams the classes k, k+8, ... (lane = column: 128-byte rows), keeping an online
// (max, sum) per column; the block combines the eight partial results, then re-streams the logits (L2) and emits / consumes
// the (T,H,N,C) side through a 32 x 32 transposing tile.  ~2x the algorithmic reads: a fallback, not the CRNN-2D path.
// =====================================================================================================
__device__ __forceinline__ void online_merge(float &m, float &s, float m2, float s2) {
    const float nm = fmaxf(m, m2);
    if (nm == -INFINITY) { m = nm; s = 0.f; return; }
    s = s * ex2f((m - nm) * kLog2e) + s2 * ex2f((m2 - nm) * kLog2e);
    m = nm;
}

template <int MODE>      // 0 = forward, 1 = backward with explicit gradient, 2 = backward with the CTC factor
__global__ void __launch_bounds__(256)
ctc2d_head_tiled_kernel(HeadGeo g, const float *__restrict__ mask_logits, const float *__restrict__ cls_logits,
                        const float *__restrict__ dlp, const float *__restrict__ gfac, const float *__restrict__ go,
                        int64_t go_stride, float tiny, float log_tiny, float *__restrict__ lp, float *__restrict__ dcls,
                        float *__restrict__ gsum) {
    __shared__ float red_m[8][32], red_s[8][32], tile[32][33];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wtiles = (g.W + 31) >> 5;
    const int wt = blockIdx.x % wtiles;
    const int h = (blockIdx.x / wtiles) % g.H;
    const int n = blockIdx.x / (wtiles * g.H);
    const int w0 = wt << 5, w = w0 + lane;
    const bool valid = w < g.W;
    const int ncol = min(32, g.W - w0);
    const int64_t HW = (int64_t)g.H * g.W;
    const float *zp = cls_logits + ((int64_t)n * g.C * g.H + h) * g.W + w;
    // pass 1: per-column (max, sum) over all classes
    float m = -INFINITY, s = 0.f;
    for (int c = warp; c < g.C; c += 8) {
        const float z = valid ? __ldg(zp + (int64_t)c * HW) : -INFINITY;
        online_merge(m, s, z, 1.f);
    }
    red_m[warp][lane] = m; red_s[warp][lane] = s;
    __syncthreads();
    m = red_m[0][lane]; s = red_s[0][lane];
    for (int k = 1; k < 8; ++k) online_merge(m, s, red_m[k][lane], red_s[k][lane]);
    const float mlog = mask_logsoftmax_col(mask_logits + (int64_t)n * HW + w, g.H, g.W, h, valid);
    const float shift = mlog - m - lg2f(s) * kLn2;            // log_probs = z + shift (before the clamp)
    const float inv = 1.f / s, maskp = ex2f(mlog * kLog2e);
    const float gout = (MODE == 2 && valid) ? __ldg(go + (int64_t)n * go_stride) : 1.f;
    const int64_t cstep_out = (int64_t)g.H * g.N * g.C;
    if (MODE == 0) {
        // pass 2: 32 classes x 32 columns at a time through the transposing tile
        for (int c0 = 0; c0 < g.C; c0 += 32) {
            for (int k = warp; k < 32; k += 8) {
                const int c = c0 + k;
                float v = 0.f;
                if (valid && c < g.C) v = fmaxf(__ldg(zp + (int64_t)c * HW) + shift, log_tiny);
                tile[k][lane] = v;
            }
            __syncthreads();
            for (int wl = warp; wl < ncol; wl += 8) {
                const int c = c0 + lane;
                if (c < g.C) lp[((int64_t)(w0 + wl) * g.H + h) * g.N * g.C + (int64_t)n * g.C + c] = tile[lane][wl];
            }
            __syncthreads();
        }
        (void)cstep_out;
    } else {
        // pass 2a: tot = sum_c g_c ; pass 2b: d z_c = g_c - p_c * tot.  The upstream rows are re-read for 2b (L2).
        float tot = 0.f;
        for (int rep = 0; rep < 2; ++rep) {
            float acc = 0.f;
            for (int c0 = 0; c0 < g.C; c0 += 32) {
                for (int wl = warp; wl < ncol; wl += 8) {     // lanes over classes: coalesced upstream rows
                    const int c = c0 + lane;
                    float u = 0.f;
                    if (c < g.C)
                        u = MODE == 2 ? __ldg(gfac + ((int64_t)(w0 + wl) * g.N + n) * g.C + c)
                                      : __ldg(dlp + (((int64_t)(w0 + wl) * g.H + h) * g.N + n) * g.C + c);
                    tile[lane][wl] = u;
                }
                __syncthreads();
                for (int k = warp; k < 32; k += 8) {          // lanes over columns
                    const int c = c0 + k;
                    if (valid && c < g.C) {
                        const float p = ex2f((__ldg(zp + (int64_t)c * HW) - m) * kLog2e) * inv;
                        const float q = p * maskp;
                        const float u = tile[k][lane];
                        const float gg = q > tiny ? (MODE == 2 ? q * u * gout : u) : 0.f;
                        if (rep == 0) acc += gg;
                        else dcls[((int64_t)n * g.C + c) * HW + (int64_t)h * g.W + w] = gg - p * tot;
                    }
                }
                __syncthreads();
            }
            if (rep == 0) {
                red_s[warp][lane] = acc;
                __syncthreads();
                tot = 0.f;
                for (int k = 0; k < 8; ++k) tot += red_s[k][lane];
                if (warp == 0 && valid) gsum[((int64_t)n * g.H + h) * g.W + w] = tot;
                __syncthreads();
            }
        }
    }
}

int pick_nt(int C, int H, int tiles, size_t *smem) {
    // samples per block: as many as keep the logits tiles within 96 KB (so that >= 2 blocks share an SM), at most 8
    auto bytes = [&](int nt) { return (size_t)nt * ((size_t)C * tiles + H) * (kTW + 1) * sizeof(float); };
    int nt = 8;
    while (nt > 1 && bytes(nt) > 96 * 1024) nt >>= 1;
    *smem = bytes(nt);
    return *smem <= 200 * 1024 ? nt : 0;
}

}  // namespace

extern "C" {

int mr_ctc2d_head_fwd_f32(const float *mask_logits, const float *cls_logits, int N, int C, int H, int W, float tiny,
                          float *log_probs, void *stream) {
    if (N < 0 || C <= 0 || H <= 0 || W <= 0 || !(tiny > 0.f)) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!mask_logits || !cls_logits || !log_probs) return MR_ERR_NULL_POINTER;
    HeadGeo g{N, C, H, W, 0};
    cudaStream_t st = (cudaStream_t)stream;
    static const bool old_only = getenv("MR_HEAD_BLOCK_TILE") != nullptr;
    const bool fits32 = (int64_t)64 * H * W * 4 < (1LL << 32) && (int64_t)H * N * C * 4 < (1LL << 32);
    if (C <= 64 && fits32 && !old_only) {
        const int64_t nslabs = (int64_t)N * H * ceil_div(W, 32);
        const int wpb = C <= 40 ? 8 : 4;
        const int64_t blocks = std::min<int64_t>(ceil_div(nslabs, wpb), (int64_t)sm_count() * 32);
        if (C == 38) ctc2d_head_fwd_warp_kernel<40, 8, 38><<<(unsigned)blocks, 256, 0, st>>>(g, mask_logits, cls_logits, logf(tiny), log_probs);   // EnglishCharset
        else if (C <= 40) ctc2d_head_fwd_warp_kernel<40, 8, 0><<<(unsigned)blocks, 256, 0, st>>>(g, mask_logits, cls_logits, logf(tiny), log_probs);
        else ctc2d_head_fwd_warp_kernel<64, 4, 0><<<(unsigned)blocks, 128, 0, st>>>(g, mask_logits, cls_logits, logf(tiny), log_probs);
        return check_launch("ctc2d_head_fwd_warp_kernel");
    }
    size_t smem;
    g.NT = pick_nt(C, H, 1, &smem);
    if (!g.NT || H > 65535 || ceil_div(N, g.NT) > 65535) {
        const int64_t blocks = (int64_t)N * H * ceil_div(W, 32);
        if (blocks > 0x7fffffffLL) return MR_ERR_UNSUPPORTED;
        ctc2d_head_tiled_kernel<0><<<(unsigned)blocks, 256, 0, st>>>(g, mask_logits, cls_logits, nullptr, nullptr, nullptr, 0, tiny,
                                                                    logf(tiny), log_probs, nullptr, nullptr);
        return check_launch("ctc2d_head_tiled_kernel");
    }
    { int rc_attr = ensure_dyn_smem((const void *)ctc2d_head_fwd_kernel, smem, "head fwd smem"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)ceil_div(W, kTW), (unsigned)H, (unsigned)ceil_div(N, g.NT));
    ctc2d_head_fwd_kernel<<<grid, kThreads, smem, st>>>(g, mask_logits, cls_logits, logf(tiny), log_probs);
    return check_launch("ctc2d_head_fwd_kernel");
}

/* Exactly one of grad_log_probs [W,H,N,C] or (gfac [W,N,C], grad_out [N] with element stride) is given. */
int mr_ctc2d_head_bwd_f32(const float *mask_logits, const float *cls_logits, const float *grad_log_probs, const float *gfac,
                          const float *grad_out, int64_t grad_out_stride, int N, int C, int H, int W, float tiny,
                          float *grad_cls_logits, float *grad_mask_logits, void *stream) {
    if (N < 0 || C <= 0 || H <= 0 || W <= 0 || !(tiny > 0.f)) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!mask_logits || !cls_logits || !grad_cls_logits || !grad_mask_logits) return MR_ERR_NULL_POINTER;
    const bool factored = grad_log_probs == nullptr;
    if (factored && (!gfac || !grad_out)) return MR_ERR_NULL_POINTER;
    HeadGeo g{N, C, H, W, 0};
    cudaStream_t st = (cudaStream_t)stream;
    static const bool old_only = getenv("MR_HEAD_BLOCK_TILE") != nullptr;
    size_t smem = 0;
    g.NT = pick_nt(C, H, 2, &smem);
    const bool tile_ok = g.NT && H <= 65535 && ceil_div(N, g.NT) <= 65535;
    const bool fits32 = (int64_t)64 * H * W * 4 < (1LL << 32) && (int64_t)H * N * C * 4 < (1LL << 32);
    if (C <= 64 && fits32 && !old_only) {
        const int64_t nslabs = (int64_t)N * (factored ? 1 : H) * ceil_div(W, 32);
        const int wpb = C <= 40 ? 8 : 4;
        const int64_t blocks = std::min<int64_t>(ceil_div(nslabs, wpb), (int64_t)sm_count() * 32);
#define MR_HEAD_BWD(CRV, FACV, WPB, CXV)                                                                                     \
        ctc2d_head_bwd_warp_kernel<CRV, FACV, WPB, CXV><<<(unsigned)blocks, WPB * 32, 0, st>>>(                                \
            g, mask_logits, cls_logits, grad_log_probs, gfac, grad_out, grad_out_stride, tiny, grad_cls_logits, grad_mask_logits)
        if (C == 38) { if (factored) MR_HEAD_BWD(40, true, 8, 38); else MR_HEAD_BWD(40, false, 8, 38); }
        else if (C <= 40) { if (factored) MR_HEAD_BWD(40, true, 8, 0); else MR_HEAD_BWD(40, false, 8, 0); }
        else { if (factored) MR_HEAD_BWD(64, true, 4, 0); else MR_HEAD_BWD(64, false, 4, 0); }
#undef MR_HEAD_BWD
    } else if (!tile_ok) {
        const int64_t blocks = (int64_t)N * H * ceil_div(W, 32);
        if (blocks > 0x7fffffffLL) return MR_ERR_UNSUPPORTED;
        if (factored)
            ctc2d_head_tiled_kernel<2><<<(unsigned)blocks, 256, 0, st>>>(g, mask_logits, cls_logits, nullptr, gfac, grad_out, grad_out_stride,
                                                                        tiny, logf(tiny), nullptr, grad_cls_logits, grad_mask_logits);
        else
            ctc2d_head_tiled_kernel<1><<<(unsigned)blocks, 256, 0, st>>>(g, mask_logits, cls_logits, grad_log_probs, nullptr, nullptr, 0,
                                                                        tiny, logf(tiny), nullptr, grad_cls_logits, grad_mask_logits);
    } else {
    {
        int rc_attr = factored ? ensure_dyn_smem((const void *)ctc2d_head_bwd_kernel<true>, smem, "head bwd smem")
                               : ensure_dyn_smem((const void *)ctc2d_head_bwd_kernel<false>, smem, "head bwd smem");
        if (rc_attr) return rc_attr;
    }
    dim3 grid((unsigned)ceil_div(W, kTW), (unsigned)H, (unsigned)ceil_div(N, g.NT));
    if (factored)
        ctc2d_head_bwd_kernel<true><<<grid, kThreads, smem, st>>>(g, mask_logits, cls_logits, nullptr, gfac, grad_out, grad_out_stride,
                                                                   tiny, grad_cls_logits, grad_mask_logits);
    else
        ctc2d_head_bwd_kernel<false><<<grid, kThreads, smem, st>>>(g, mask_logits, cls_logits, grad_log_probs, nullptr, nullptr, 0,
                                                                    tiny, grad_cls_logits, grad_mask_logits);
    }
    int rc = check_launch("ctc2d_head_bwd_kernel");
    if (rc) return rc;
    const int64_t cols = (int64_t)N * W;
    ctc2d_head_mask_bwd_kernel<<<(unsigned)ceil_div(cols, 256), 256, 0, st>>>(N, H, W, mask_logits, grad_mask_logits);
    return check_launch("ctc2d_head_mask_bwd_kernel");
}

}  // extern "C"
