// CRNN stem (backbones/crnn.py layer 0): Conv2d(3, 64, 3, 1, 1) -> ReLU -> MaxPool2d(2, 2), forward and weight gradient,
// each as one kernel over the NCHW fp32 input image.  No im2col matrix, conv output or conv-output gradient reaches HBM:
// the forward reads x and writes the pooled NHWC bf16 activation (and one routing byte per pooled value), the backward
// reads x, dy and the routing bytes and writes one fp32 partial row per CTA.
//
// Tiles.  A CTA owns TH = 8 conv rows x TW = 64 conv columns (4 x 32 pooled outputs) and stages its input halo (10 x 66
// pixels) in shared memory, rounded to bf16 exactly as mr_nchw_to_nhwc rounds it.  A warp unit is 2 conv rows x 16 conv
// columns = 8 pooled outputs; each CTA's 4 warps take 4 units each.  Both GEMMs run on mma.sync m16n8k16 bf16 with fp32
// accumulation.
//
// Forward: M = conv pixels, N = 64 output channels, K = (kh, kw, c4): the input is staged [row][col][4 channels], so one
// kernel row of a pixel's patch is 12 contiguous bf16 and one k16 step per kernel row covers it (columns 12..15 are zero).
// M rows g / g+8 of m-tile 0 are the pixels (h, 2g) / (h+1, 2g) of the unit and m-tile 1 the same one column to the right,
// so every thread holds all four values of its 2x2 pooling windows in its accumulator fragments.  The epilogue keeps the
// rounding sequence of the unfused path (z = bf16(conv), a = bf16(max(z + bias, 0))), takes the first arg-max with a
// strict '>' from -inf in (i, j) order and stores y through a per-warp staging buffer as 16-byte rows.
//
// Routing byte: i * 2 + j of the arg-max when the pooled value is > 0, else kNotPositive.  The backward needs nothing else:
// dz(h, w) = dy(h/2, w/2) where the byte names (h, w), 0 elsewhere.
//
// Backward: M = output channels (row g of m-tile mt is channel 16 mt + 2g, row g+8 channel 16 mt + 2g + 1, so one 32-bit
// load of dy feeds both), N = reference weight columns c * 9 + kh * 3 + kw (27 of them) plus a column of ones at 27 that
// makes the conv-bias gradient a by-product, K = 16 consecutive conv pixels of one row.  The input is staged planar
// [c][row][col] twice, the second copy shifted by one column, so that a pixel pair (w, w+1) with w even is one aligned
// 32-bit load for every tap.  Each CTA walks tiles with a fixed grid stride, adds its warps' accumulators in a fixed order
// and stores one row of [64 * 27 weight | 64 bias] partials; partials_finalize_kernel adds the rows in double.  Two runs
// give the same bits.
#include "common.cuh"
#include <cuda_bf16.h>
#include <algorithm>

namespace {
using namespace mr;

constexpr int kCout = 64;
constexpr int TH = 8, TW = 64;                     // conv rows / columns per CTA tile
constexpr int SR = TH + 2, SC = TW + 2;            // staged input rows / columns (1-pixel halo)
constexpr int kWarps = 4, kThreads = kWarps * 32;
constexpr int kUnits = (TH / 2) * (TW / 16);       // warp units per tile
constexpr unsigned char kNotPositive = 4;          // routing byte of a pooled value that fails ReLU'
constexpr int kWCols = 27;                         // reference weight columns c * 9 + kh * 3 + kw
constexpr int kPartCols = kCout * kWCols + kCout;  // partial row: dW [64][27] then dbias [64]

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t *>(&v);
}

__device__ __forceinline__ void mma_bf16(float *d, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

struct StemGeo {
    int N, H, W, Hp, Wp, tiles_h, tiles_w;
    int64_t tiles;
};

__device__ __forceinline__ float bf16r(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
__device__ __forceinline__ float fmax_nan(float a, float b) {      // max that returns NaN if either operand is NaN
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// ------------------------------------------------------------------------------------------------ forward
// staged input: [SR][SC][4] bf16, channel 3 zero; staged (r, s) is input pixel (h0 - 1 + r, w0 - 1 + s), zero outside
__global__ void __launch_bounds__(kThreads, 3)
crnn_stem_fwd_kernel(StemGeo g, const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bias,
                     __nv_bfloat16 *__restrict__ y, unsigned char *__restrict__ idx) {
    __shared__ __align__(16) uint2 xs[SR * SC];
    __shared__ __align__(16) unsigned char ys[kWarps][8 * 144];          // 8 pooled pixels x 128 B, row pitch 144 B
    __shared__ __align__(16) unsigned char is[kWarps][8 * 80];           // 8 pooled pixels x 64 B, row pitch 80 B
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gq = lane >> 2, tq = lane & 3;

    // B fragments (weights, bf16-rounded like the GEMM operand of the unfused path): k-step kh, n-tile nt
    uint32_t bw[3][8][2];
#pragma unroll
    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const float *wc = w + (nt * 8 + gq) * 27 + kh * 3;              // [cout][c][kh][kw]
            float v[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) {                                  // k = 2t + (r & 1) + 8 (r >> 1)
                const int k = 2 * tq + (r & 1) + 8 * (r >> 1);
                const int kw = k >> 2, c = k & 3;
                v[r] = (k < 12 && c < 3) ? __ldg(wc + c * 9 + kw) : 0.f;
            }
            bw[kh][nt][0] = pack_bf16(v[0], v[1]);
            bw[kh][nt][1] = pack_bf16(v[2], v[3]);
        }

    const int64_t plane = (int64_t)g.H * g.W;
    for (int64_t tile = blockIdx.x; tile < g.tiles; tile += gridDim.x) {
        const int n = (int)(tile / (g.tiles_h * g.tiles_w));
        const int rem = (int)(tile - (int64_t)n * g.tiles_h * g.tiles_w);
        const int h0 = (rem / g.tiles_w) * TH, w0 = (rem % g.tiles_w) * TW;
        const float *xn = x + (int64_t)n * 3 * plane;
        __syncthreads();                                                   // previous tile's readers are done
        constexpr int kPer = (SR * SC + kThreads - 1) / kThreads;
        float v[kPer][3];
#pragma unroll
        for (int u = 0; u < kPer; ++u) {
            const int i = threadIdx.x + u * kThreads;
            const int r = i / SC, s = i - r * SC;
            const int h = h0 - 1 + r, ww = w0 - 1 + s;
            const bool ok = i < SR * SC && h >= 0 && h < g.H && ww >= 0 && ww < g.W;
#pragma unroll
            for (int c = 0; c < 3; ++c) v[u][c] = ok ? __ldg(xn + c * plane + (int64_t)h * g.W + ww) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < kPer; ++u) {
            const int i = threadIdx.x + u * kThreads;
            if (i < SR * SC) xs[i] = make_uint2(pack_bf16(v[u][0], v[u][1]), pack_bf16(v[u][2], 0.f));
        }
        __syncthreads();

        for (int unit = warp; unit < kUnits; unit += kWarps) {
            const int rp = unit / (TW / 16), cu = unit % (TW / 16);
            const int hp = (h0 >> 1) + rp, wp0 = (w0 >> 1) + cu * 8;
            if (hp >= g.Hp || wp0 >= g.Wp) continue;                      // warp-uniform
            float acc[2][8][4];
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) acc[m][nt][e] = 0.f;
            // conv pixel (2 rp + dr, 16 cu + 2 gq + m) of the tile; its kernel-row-kh patch starts at staged (2 rp + dr + kh, 16 cu + 2 gq + m)
            const unsigned char *base = reinterpret_cast<const unsigned char *>(xs) + ((2 * rp) * SC + 16 * cu + 2 * gq) * 8;
#pragma unroll
            for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
                for (int m = 0; m < 2; ++m) {
                    const unsigned char *p0 = base + (kh * SC + m) * 8, *p1 = p0 + SC * 8;
                    const uint32_t a0 = *reinterpret_cast<const uint32_t *>(p0 + 4 * tq);
                    const uint32_t a1 = *reinterpret_cast<const uint32_t *>(p1 + 4 * tq);
                    const uint32_t a2 = tq < 2 ? *reinterpret_cast<const uint32_t *>(p0 + 16 + 4 * tq) : 0u;
                    const uint32_t a3 = tq < 2 ? *reinterpret_cast<const uint32_t *>(p1 + 16 + 4 * tq) : 0u;
#pragma unroll
                    for (int nt = 0; nt < 8; ++nt) mma_bf16(acc[m][nt], a0, a1, a2, a3, bw[kh][nt][0], bw[kh][nt][1]);
                }
            }
            // epilogue: window (i, j) = (0,0) acc[0][.][e], (0,1) acc[1][.][e], (1,0) acc[0][.][2+e], (1,1) acc[1][.][2+e]
            unsigned char *yw = ys[warp], *iw = is[warp];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const int co = nt * 8 + 2 * tq;
                float best[2];
                unsigned char bi[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float b = __ldg(bias + co + e);
                    const float win[4] = {acc[0][nt][e], acc[1][nt][e], acc[0][nt][2 + e], acc[1][nt][2 + e]};
                    best[e] = -INFINITY;
                    bi[e] = 0;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {       // ReLU and max keep a NaN, as ATen's relu and max_pool2d do
                        const float a = bf16r(fmax_nan(bf16r(win[k]) + b, 0.f));
                        if (!(a <= best[e])) bi[e] = (unsigned char)k;
                        best[e] = fmax_nan(best[e], a);
                    }
                    if (!(best[e] > 0.f)) bi[e] = kNotPositive;
                }
                *reinterpret_cast<uint32_t *>(yw + gq * 144 + co * 2) = pack_bf16(best[0], best[1]);
                *reinterpret_cast<uint16_t *>(iw + gq * 80 + co) = (uint16_t)(bi[0] | (bi[1] << 8));
            }
            __syncwarp();
            const int nv = min(8, g.Wp - wp0);
            const int64_t o = ((int64_t)n * g.Hp + hp) * g.Wp + wp0;           // first pooled pixel of the unit
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int q = lane + 32 * u, px = q >> 3;                         // 8 16-byte chunks per pixel
                if (px < nv)
                    __stcs(reinterpret_cast<uint4 *>(y + (o + px) * kCout) + (q & 7),
                           *reinterpret_cast<const uint4 *>(yw + px * 144 + (q & 7) * 16));
            }
            if (idx) {
                const int px = lane >> 2;                                         // 4 16-byte chunks per pixel
                if (px < nv)
                    __stcs(reinterpret_cast<uint4 *>(idx + (o + px) * kCout) + (lane & 3),
                           *reinterpret_cast<const uint4 *>(iw + px * 80 + (lane & 3) * 16));
            }
            __syncwarp();
        }
    }
}

// ------------------------------------------------------------------------------------------------ backward
// staged input: planar [2 copies][3][SR][SP] bf16; copy 1 is copy 0 shifted left by one column
constexpr int SP = SC + 2;                         // even row pitch (32-bit pixel-pair loads)
constexpr int kPlane = SR * SP;

__global__ void __launch_bounds__(kThreads, 3)
crnn_stem_bwd_kernel(StemGeo g, const float *__restrict__ x, const __nv_bfloat16 *__restrict__ dy,
                     const unsigned char *__restrict__ idx, float *__restrict__ part) {
    __shared__ __align__(16) __nv_bfloat16 xs[2 * 3 * kPlane];
    __shared__ float red[kWarps][kCout][33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gq = lane >> 2, tq = lane & 3;

    // per n-tile: staged offset (elements) of this lane's weight column k = 8 nt + gq, or -1 for the ones column / unused
    int boff[4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        const int k = nt * 8 + gq;
        const int c = k / 9, kh = (k % 9) / 3, kw = k % 3;
        boff[nt] = k < kWCols ? (kw & 1) * 3 * kPlane + c * kPlane + kh * SP + (kw & 2) : -1;
    }
    float acc[4][4][4];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;

    const int64_t plane = (int64_t)g.H * g.W;
    for (int64_t tile = blockIdx.x; tile < g.tiles; tile += gridDim.x) {
        const int n = (int)(tile / (g.tiles_h * g.tiles_w));
        const int rem = (int)(tile - (int64_t)n * g.tiles_h * g.tiles_w);
        const int h0 = (rem / g.tiles_w) * TH, w0 = (rem % g.tiles_w) * TW;
        const float *xn = x + (int64_t)n * 3 * plane;
        __syncthreads();
        constexpr int kPer = 8;                                            // loads in flight per thread
#pragma unroll 1
        for (int i0 = 0; i0 < 3 * kPlane; i0 += kPer * kThreads) {
            float v[kPer];
#pragma unroll
            for (int u = 0; u < kPer; ++u) {
                const int i = i0 + threadIdx.x + u * kThreads;
                const int c = i / kPlane, r = (i % kPlane) / SP, s = i % SP;
                const int h = h0 - 1 + r, ww = w0 - 1 + s;
                const bool ok = i < 3 * kPlane && h >= 0 && h < g.H && ww >= 0 && ww < g.W;
                v[u] = ok ? __ldg(xn + c * plane + (int64_t)h * g.W + ww) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < kPer; ++u) {
                const int i = i0 + threadIdx.x + u * kThreads;
                if (i < 3 * kPlane) {
                    const __nv_bfloat16 b = __float2bfloat16_rn(v[u]);
                    xs[i] = b;
                    if (i % SP) xs[3 * kPlane + i - 1] = b;              // copy 1: column s - 1
                }
            }
        }
        __syncthreads();

        for (int unit = warp; unit < kUnits; unit += kWarps) {
            const int rp = unit / (TW / 16), cu = unit % (TW / 16);
            const int hp = (h0 >> 1) + rp, wpb = (w0 >> 1) + cu * 8;
            if (hp >= g.Hp || wpb >= g.Wp) continue;                      // warp-uniform
            // dy / routing of pooled pixels wpb + tq (conv columns 2 tq, 2 tq + 1) and wpb + 4 + tq (8 + 2 tq, 9 + 2 tq),
            // output channels 16 mt + 2 gq and 16 mt + 2 gq + 1
            uint32_t dv[2][4];
            uint16_t rv[2][4];
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int wp = wpb + 4 * hf + tq;
                const bool ok = wp < g.Wp;
                const int64_t q = (((int64_t)n * g.Hp + hp) * g.Wp + wp) * kCout + 2 * gq;
#pragma unroll
                for (int mt = 0; mt < 4; ++mt) {
                    dv[hf][mt] = ok ? __ldg(reinterpret_cast<const unsigned *>(dy + q + 16 * mt)) : 0u;
                    rv[hf][mt] = ok ? __ldg(reinterpret_cast<const unsigned short *>(idx + q + 16 * mt))
                                    : (uint16_t)(kNotPositive | (kNotPositive << 8));
                }
            }
#pragma unroll
            for (int dr = 0; dr < 2; ++dr) {
                // B: pixel pair (conv columns 2 tq, 2 tq + 1) / (8 + 2 tq, 9 + 2 tq) of conv row 2 rp + dr, column k
                const int pix = (2 * rp + dr) * SP + 16 * cu + 2 * tq;
                uint32_t b[4][2];
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    if (boff[nt] >= 0) {
                        b[nt][0] = *reinterpret_cast<const uint32_t *>(xs + boff[nt] + pix);
                        b[nt][1] = *reinterpret_cast<const uint32_t *>(xs + boff[nt] + pix + 8);
                    } else {
                        b[nt][0] = b[nt][1] = (nt * 8 + gq == kWCols) ? 0x3F803F80u : 0u;   // ones: dbias column
                    }
                }
#pragma unroll
                for (int mt = 0; mt < 4; ++mt) {
                    uint32_t a[4];
#pragma unroll
                    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {                           // e: channel 16 mt + 2 gq + e
                            const uint32_t d = (dv[hf][mt] >> (16 * e)) & 0xFFFFu;
                            const unsigned r = (rv[hf][mt] >> (8 * e)) & 0xFFu;
                            a[2 * hf + e] = (r == 2u * dr ? d : 0u) | (r == 2u * dr + 1u ? d << 16 : 0u);
                        }
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) mma_bf16(acc[mt][nt], a[0], a[1], a[2], a[3], b[nt][0], b[nt][1]);
                }
            }
        }
    }
    // accumulator (row g / g+8 of m-tile mt = channel 16 mt + 2 gq / + 1, column 8 nt + 2 tq + {0,1}) -> red, then the
    // warps are added in a fixed order
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e)
                red[warp][16 * mt + 2 * gq + (e >> 1)][8 * nt + 2 * tq + (e & 1)] = acc[mt][nt][e];
    __syncthreads();
    float *row = part + (int64_t)blockIdx.x * kPartCols;
    for (int i = threadIdx.x; i < kCout * (kWCols + 1); i += kThreads) {
        const int co = i / (kWCols + 1), k = i % (kWCols + 1);
        float s = 0.f;
#pragma unroll
        for (int wi = 0; wi < kWarps; ++wi) s += red[wi][co][k];
        row[k < kWCols ? co * kWCols + k : kCout * kWCols + co] = s;
    }
}

__global__ void stem_grads_kernel(const double *__restrict__ sums, float *__restrict__ dw, float *__restrict__ dbias) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < kCout * kWCols) dw[i] = (float)sums[i];
    else if (i < kPartCols) dbias[i - kCout * kWCols] = (float)sums[i];
}

// shapes and the geometry the stem covers: Conv2d(3, 64, 3, stride 1, padding 1) + MaxPool2d(2, 2, 0), H, W >= 2
int stem_geo(StemGeo &g, int N, int Cin, int H, int W, int Cout, int kh, int kw, int sh, int sw, int ph, int pw, int pkh,
             int pkw, int psh, int psw, int pph, int ppw) {
    if (N < 0 || Cin <= 0 || H <= 0 || W <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || ph < 0 ||
        pw < 0 || pkh <= 0 || pkw <= 0 || psh <= 0 || psw <= 0 || pph < 0 || ppw < 0)
        return MR_ERR_BAD_SHAPE;
    if (Cin != 3 || Cout != kCout || kh != 3 || kw != 3 || sh != 1 || sw != 1 || ph != 1 || pw != 1 || pkh != 2 ||
        pkw != 2 || psh != 2 || psw != 2 || pph != 0 || ppw != 0 || H < 2 || W < 2)
        return MR_ERR_UNSUPPORTED;
    g.N = N; g.H = H; g.W = W; g.Hp = H / 2; g.Wp = W / 2;
    g.tiles_h = (int)ceil_div(g.Hp, TH / 2);
    g.tiles_w = (int)ceil_div(g.Wp, TW / 2);
    g.tiles = (int64_t)N * g.tiles_h * g.tiles_w;
    return MR_OK;
}

}  // namespace

extern "C" {

int mr_crnn_stem_fwd(const float *x, const float *w, const float *bias, int N, int Cin, int H, int W, int Cout, int kh,
                     int kw, int sh, int sw, int ph, int pw, int pkh, int pkw, int psh, int psw, int pph, int ppw, void *y,
                     unsigned char *idx, void *stream) {
    StemGeo g;
    int rc = stem_geo(g, N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, pkh, pkw, psh, psw, pph, ppw);
    if (rc) return rc;
    if (N == 0) return MR_OK;
    if (!x || !w || !bias || !y) return MR_ERR_NULL_POINTER;
    const int64_t blocks = std::min<int64_t>(g.tiles, (int64_t)sm_count() * 3 * 16);
    crnn_stem_fwd_kernel<<<(int)blocks, kThreads, 0, (cudaStream_t)stream>>>(g, x, w, bias, (__nv_bfloat16 *)y, idx);
    return check_launch("crnn_stem_fwd_kernel");
}

int mr_crnn_stem_bwd(const float *x, const void *dy, const unsigned char *idx, int N, int Cin, int H, int W, int Cout,
                     int kh, int kw, int sh, int sw, int ph, int pw, int pkh, int pkw, int psh, int psw, int pph, int ppw,
                     float *dw, float *dbias, double *sums, void *stream) {
    StemGeo g;
    int rc = stem_geo(g, N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, pkh, pkw, psh, psw, pph, ppw);
    if (rc) return rc;
    if (!dw || !dbias || !sums) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) {
        MR_CUDA_TRY(cudaMemsetAsync(dw, 0, sizeof(float) * kCout * kWCols, st), "memset dw");
        MR_CUDA_TRY(cudaMemsetAsync(dbias, 0, sizeof(float) * kCout, st), "memset dbias");
        return MR_OK;
    }
    if (!x || !dy || !idx) return MR_ERR_NULL_POINTER;
    int nb = (int)std::min<int64_t>(g.tiles, (int64_t)sm_count() * 3);
    float *part = block_partials(nb, kPartCols);
    if (!part) return MR_ERR_CUDA;
    crnn_stem_bwd_kernel<<<nb, kThreads, 0, st>>>(g, x, (const __nv_bfloat16 *)dy, idx, part);
    rc = check_launch("crnn_stem_bwd_kernel");
    if (rc) return rc;
    rc = finalize_partials(part, nb, kPartCols, sums, st);
    if (rc) return rc;
    stem_grads_kernel<<<(int)ceil_div(kPartCols, 256), 256, 0, st>>>(sums, dw, dbias);
    return check_launch("stem_grads_kernel");
}

}  // extern "C"
