// NHWC building blocks of the CRNN training engine (sm_90a): layout conversion, im2col / col2im, fused
// bias+ReLU+max-pool (forward and backward), training-mode BatchNorm (stats / apply / backward), column sums,
// LSTM cell (forward / backward), fused Adam, weight layout packs, greedy CTC decoders.  All HBM-bound streaming
// kernels: 16-byte vector accesses along the channel dimension, fp32 accumulation; per-channel sums leave each block
// as one row of an fp32 partial buffer and are added in double by a small second kernel (no atomics on the hot path).
//
// Why these exist: with the ATen/cuDNN composition of the reference's modules (backbones/crnn.py:46-55,
// decoders/crnn.py:8-24) the tensor-core convolutions are a small part of a training step; NCHW max-pool forward /
// backward, NCHW<->NHWC transposes, BatchNorm and the per-timestep LSTM glue are most of it.  Keeping activations NHWC end to end and fusing the elementwise chains
// removes that traffic.
//
// dtype codes: 0 = float32, 1 = bfloat16.  "rows" = N*H*W pixels, C = channels (innermost).
#include "common.cuh"
#include <cuda_bf16.h>
#include <math.h>
#include <algorithm>
#include <string.h>

namespace {
using namespace mr;
typedef __nv_bfloat16 bf16;

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<bf16>(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16_rn(v); }

// 16-byte vector of T
template <typename T> struct Vec16 { static constexpr int N = 16 / sizeof(T); uint4 raw; };
template <typename T> __device__ __forceinline__ void unpack(const uint4 &r, float *f) {
    constexpr int N = 16 / sizeof(T);
    const T *p = reinterpret_cast<const T *>(&r);
#pragma unroll
    for (int i = 0; i < N; ++i) f[i] = to_f<T>(p[i]);
}
template <typename T> __device__ __forceinline__ uint4 pack(const float *f) {
    constexpr int N = 16 / sizeof(T);
    uint4 r;
    T *p = reinterpret_cast<T *>(&r);
#pragma unroll
    for (int i = 0; i < N; ++i) p[i] = from_f<T>(f[i]);
    return r;
}

template <int VN> __device__ __forceinline__ void store_bytes(unsigned char *dst, const unsigned char *b);
template <> __device__ __forceinline__ void store_bytes<8>(unsigned char *dst, const unsigned char *b) {
    uint2 v; memcpy(&v, b, 8); *reinterpret_cast<uint2 *>(dst) = v;
}
template <> __device__ __forceinline__ void store_bytes<4>(unsigned char *dst, const unsigned char *b) {
    unsigned v; memcpy(&v, b, 4); *reinterpret_cast<unsigned *>(dst) = v;
}
template <int VN> __device__ __forceinline__ void load_bytes(const unsigned char *src, unsigned char *b);
template <> __device__ __forceinline__ void load_bytes<8>(const unsigned char *src, unsigned char *b) {
    const uint2 v = __ldg(reinterpret_cast<const uint2 *>(src)); memcpy(b, &v, 8);
}
template <> __device__ __forceinline__ void load_bytes<4>(const unsigned char *src, unsigned char *b) {
    const unsigned v = __ldg(reinterpret_cast<const unsigned *>(src)); memcpy(b, &v, 4);
}

// per-channel sums of values each thread accumulated for its (fixed) channel vector: block reduce, fp64 atomics
template <int VN>
__device__ __forceinline__ void block_channel_sum(const float *acc, int cv, double *sums, float (*red)[VN + 1]) {
#pragma unroll
    for (int e = 0; e < VN; ++e) red[threadIdx.x][e] = acc[e];
    __syncthreads();
    if ((int)threadIdx.x < cv) {
        const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
        const int cvec = (int)(gtid % cv);
#pragma unroll
        for (int e = 0; e < VN; ++e) {
            float t = 0.f;
            for (int k = threadIdx.x; k < (int)blockDim.x; k += cv) t += red[k][e];
            atomicAdd(sums + cvec * VN + e, (double)t);
        }
    }
}

// Same reduction without atomics: every block stores its per-channel sums as one row of a [gridDim.x, C] fp32 scratch;
// partials_finalize_kernel adds the rows in double.  (fp64 atomics from thousands of blocks onto C addresses serialise
// and cost more than the streaming itself.)
template <int VN>
__device__ __forceinline__ void block_channel_partial(const float *acc, int cv, float *part_row, float (*red)[VN + 1]) {
#pragma unroll
    for (int e = 0; e < VN; ++e) red[threadIdx.x][e] = acc[e];
    __syncthreads();
    if ((int)threadIdx.x < cv) {
        const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
        const int cvec = (int)(gtid % cv);
#pragma unroll
        for (int e = 0; e < VN; ++e) {
            float t = 0.f;
            for (int k = threadIdx.x; k < (int)blockDim.x; k += cv) t += red[k][e];
            part_row[cvec * VN + e] = t;
        }
    }
}

// out[c] = sum_b part[b, c] (double).  Block = 32 columns x 32 row lanes: each lane walks rows lane, lane+32, ... with
// four loads in flight (a one-thread-per-column loop over ~1000 rows is one long latency chain), then a shared-memory
// reduction over the lanes.
__global__ void __launch_bounds__(1024)
partials_finalize_kernel(const float *__restrict__ part, int nb, int ncols, double *__restrict__ out) {
    __shared__ double red[32][33];
    const int cx = threadIdx.x, ry = threadIdx.y;
    const int c = blockIdx.x * 32 + cx;
    double a0 = 0, a1 = 0, a2 = 0, a3 = 0;
    if (c < ncols) {
        int b = ry;
        for (; b + 96 < nb; b += 128) {
            const float v0 = part[(int64_t)b * ncols + c], v1 = part[(int64_t)(b + 32) * ncols + c];
            const float v2 = part[(int64_t)(b + 64) * ncols + c], v3 = part[(int64_t)(b + 96) * ncols + c];
            a0 += v0; a1 += v1; a2 += v2; a3 += v3;
        }
        for (; b < nb; b += 32) a0 += part[(int64_t)b * ncols + c];
    }
    red[ry][cx] = (a0 + a1) + (a2 + a3);
    __syncthreads();
    if (ry == 0 && c < ncols) {
        double t = 0;
#pragma unroll
        for (int k = 0; k < 32; ++k) t += red[k][cx];
        out[c] = t;
    }
}

constexpr int kMaxPartialBlocks = 132 * 8;        // sizes a scratch buffer: 8 blocks per SM of an H100 SXM
constexpr int kMaxPartialCols = 4096;     // 2 * C columns of statistics for C up to 2048 (ResNet-50 layer4)
// Library-owned scratch for the block partial sums (stream-ordered use on one stream at a time).  Allocated on first
// use, which must not happen inside a CUDA-graph capture: callers run one eager step before capturing (as they must
// for cuBLAS anyway).  NULL when the allocation is impossible -> the fp64-atomic path is used instead.
float *partials_scratch() {
    static float *buf[16] = {nullptr};                    // one scratch per DEVICE (a process may drive several GPUs)
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return nullptr;
    if (!buf[dev]) {
        void *p = nullptr;
        if (cudaMalloc(&p, sizeof(float) * (size_t)kMaxPartialBlocks * kMaxPartialCols) == cudaSuccess) buf[dev] = (float *)p;
        else cudaGetLastError();                          // e.g. called under capture: retry on the next eager call
    }
    return buf[dev];
}

inline int grid1d(int64_t work, int block, int per_sm = 16) {
    int64_t b = ceil_div(work, block);
    const int64_t cap = (int64_t)sm_count() * per_sm;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// ---------------------------------------------------------------- NCHW fp32 -> NHWC (channel-padded) T
template <typename T>
__global__ void nchw_to_nhwc_kernel(const float *__restrict__ x, int N, int C, int HW, int Cp, T *__restrict__ y) {
    const int64_t total = (int64_t)N * HW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n = i / HW;
        const int64_t p = i - n * HW;
        const float *src = x + n * C * HW + p;
        T *dst = y + i * Cp;
        for (int c = 0; c < Cp; ++c) dst[c] = from_f<T>(c < C ? src[(int64_t)c * HW] : 0.f);
    }
}

// NHWC T [rows, C] -> NCHW fp32 (used for the gradient w.r.t. the input image and generic layout exits)
template <typename T>
__global__ void nhwc_to_nchw_kernel(const T *__restrict__ x, int N, int C, int HW, int Cp, float *__restrict__ y) {
    const int64_t total = (int64_t)N * C * HW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = i % HW;
        const int64_t nc = i / HW;
        const int64_t n = nc / C, c = nc - n * C;
        y[i] = to_f<T>(x[(n * HW + p) * Cp + c]);
    }
}

// ---------------------------------------------------------------- im2col / col2im (stride 1)
struct ConvGeo { int N, H, W, C, kh, kw, ph, pw, Ho, Wo, K, Kp; };

// col[p][(i*kw + j)*C + c] = x[n, ho+i-ph, wo+j-pw, c]  (0 outside), columns K..Kp zero.  Vector path: C % VN == 0.
template <typename T>
__global__ void im2col_vec_kernel(ConvGeo g, const T *__restrict__ x, T *__restrict__ col) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = g.C / VN;                       // vectors per tap
    const int kvec = g.Kp / VN;                    // vectors per column row
    const int64_t total = (int64_t)g.N * g.Ho * g.Wo * kvec;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int kv = (int)(idx % kvec);
        const int64_t p = idx / kvec;
        const int wo = (int)(p % g.Wo);
        const int64_t r = p / g.Wo;
        const int ho = (int)(r % g.Ho);
        const int n = (int)(r / g.Ho);
        uint4 v = make_uint4(0, 0, 0, 0);
        const int tap = kv / cv;
        if (tap < g.kh * g.kw) {
            const int c0 = (kv - tap * cv) * VN;
            const int i = tap / g.kw, j = tap - i * g.kw;
            const int h = ho + i - g.ph, w = wo + j - g.pw;
            if (h >= 0 && h < g.H && w >= 0 && w < g.W)
                v = __ldg(reinterpret_cast<const uint4 *>(x + (((int64_t)n * g.H + h) * g.W + w) * g.C + c0));
        }
        reinterpret_cast<uint4 *>(col)[idx] = v;
    }
}
template <typename T>
__global__ void im2col_scalar_kernel(ConvGeo g, const T *__restrict__ x, T *__restrict__ col) {
    const int64_t total = (int64_t)g.N * g.Ho * g.Wo * g.Kp;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(idx % g.Kp);
        const int64_t p = idx / g.Kp;
        const int wo = (int)(p % g.Wo);
        const int64_t r = p / g.Wo;
        const int ho = (int)(r % g.Ho);
        const int n = (int)(r / g.Ho);
        T v = from_f<T>(0.f);
        if (k < g.K) {
            const int tap = k / g.C, c = k - tap * g.C;
            const int i = tap / g.kw, j = tap - i * g.kw;
            const int h = ho + i - g.ph, w = wo + j - g.pw;
            if (h >= 0 && h < g.H && w >= 0 && w < g.W) v = x[(((int64_t)n * g.H + h) * g.W + w) * g.C + c];
        }
        col[idx] = v;
    }
}

// dx[n,h,w,c] = sum_{i,j} dcol[(n, h-i+ph, w-j+pw)][(i*kw+j)*C + c]   (gather form, no atomics)
template <typename T>
__global__ void col2im_vec_kernel(ConvGeo g, const T *__restrict__ dcol, T *__restrict__ dx) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = g.C / VN;
    const int64_t total = (int64_t)g.N * g.H * g.W * cv;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int c0 = (int)(idx % cv) * VN;
        const int64_t p = idx / cv;
        const int w = (int)(p % g.W);
        const int64_t r = p / g.W;
        const int h = (int)(r % g.H);
        const int n = (int)(r / g.H);
        float acc[VN];
#pragma unroll
        for (int e = 0; e < VN; ++e) acc[e] = 0.f;
        for (int i = 0; i < g.kh; ++i) {
            const int ho = h - i + g.ph;
            if (ho < 0 || ho >= g.Ho) continue;
            for (int j = 0; j < g.kw; ++j) {
                const int wo = w - j + g.pw;
                if (wo < 0 || wo >= g.Wo) continue;
                const uint4 v = __ldg(reinterpret_cast<const uint4 *>(
                    dcol + (((int64_t)n * g.Ho + ho) * g.Wo + wo) * g.Kp + (i * g.kw + j) * g.C + c0));
                float f[VN];
                unpack<T>(v, f);
#pragma unroll
                for (int e = 0; e < VN; ++e) acc[e] += f[e];
            }
        }
        reinterpret_cast<uint4 *>(dx)[idx] = pack<T>(acc);
    }
}

// ---------------------------------------------------------------- bias + ReLU (+ max-pool) on a GEMM output
struct PoolGeo { int N, H, W, C, kh, kw, sh, sw, ph, pw, Ho, Wo; };

// y[n,ho,wo,c] = max over window of relu(x + bias) ; idx = first arg-max in (i,j) scan order (ATen's strict '>').
// Padded positions never win (ATen pads with -inf).  x is the raw GEMM output [N*H*W, C].
template <typename T>
__global__ void bias_relu_pool_fwd_kernel(PoolGeo g, const T *__restrict__ x, const float *__restrict__ bias,
                                          T *__restrict__ y, unsigned char *__restrict__ idx) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = g.C / VN;
    const int64_t total = (int64_t)g.N * g.Ho * g.Wo * cv;
    float bb[VN];
    int c_cached = -1;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int c0 = (int)(t % cv) * VN;
        if (c0 != c_cached) {          // invariant across the grid-stride loop when cv divides the block size
#pragma unroll
            for (int e = 0; e < VN; ++e) bb[e] = bias[c0 + e];
            c_cached = c0;
        }
        const int64_t p = t / cv;
        const int wo = (int)(p % g.Wo);
        const int64_t r = p / g.Wo;
        const int ho = (int)(r % g.Ho);
        const int n = (int)(r / g.Ho);
        float best[VN];
        int bi[VN];
#pragma unroll
        for (int e = 0; e < VN; ++e) { best[e] = -INFINITY; bi[e] = 0; }
        for (int i = 0; i < g.kh; ++i) {
            const int h = ho * g.sh - g.ph + i;
            if (h < 0 || h >= g.H) continue;
            for (int j = 0; j < g.kw; ++j) {
                const int w = wo * g.sw - g.pw + j;
                if (w < 0 || w >= g.W) continue;
                const uint4 v = __ldg(reinterpret_cast<const uint4 *>(x + (((int64_t)n * g.H + h) * g.W + w) * g.C + c0));
                float f[VN];
                unpack<T>(v, f);
#pragma unroll
                for (int e = 0; e < VN; ++e) {
                    // round through T so that the compared values are what an unfused bias+ReLU would have stored
                    const float a = to_f<T>(from_f<T>(fmaxf(f[e] + bb[e], 0.f)));
                    if (a > best[e]) { best[e] = a; bi[e] = i * g.kw + j; }
                }
            }
        }
        reinterpret_cast<uint4 *>(y)[t] = pack<T>(best);
        unsigned char ib[VN];
#pragma unroll
        for (int e = 0; e < VN; ++e) ib[e] = (unsigned char)bi[e];
        store_bytes<VN>(idx + t * VN, ib);
    }
}

// dz[n,h,w,c] (gradient w.r.t. the raw GEMM output) = sum over windows that contain (h,w) whose arg-max is (h,w)
// and whose pooled value is > 0 (ReLU') of dy[window].
template <typename T>
__global__ void __launch_bounds__(256)
bias_relu_pool_bwd_kernel(PoolGeo g, const T *__restrict__ dy, const T *__restrict__ y,
                          const unsigned char *__restrict__ idx, T *__restrict__ dz, double *__restrict__ bias_sums,
                          float *__restrict__ part) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = g.C / VN;
    const int64_t total = (int64_t)g.N * g.H * g.W * cv;
    float bsum[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) bsum[e] = 0.f;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int c0 = (int)(t % cv) * VN;
        const int64_t p = t / cv;
        const int w = (int)(p % g.W);
        const int64_t r = p / g.W;
        const int h = (int)(r % g.H);
        const int n = (int)(r / g.H);
        float acc[VN];
#pragma unroll
        for (int e = 0; e < VN; ++e) acc[e] = 0.f;
        for (int i = 0; i < g.kh; ++i) {
            const int hn = h + g.ph - i;
            if (hn < 0 || hn % g.sh) continue;
            const int ho = hn / g.sh;
            if (ho >= g.Ho) continue;
            for (int j = 0; j < g.kw; ++j) {
                const int wn = w + g.pw - j;
                if (wn < 0 || wn % g.sw) continue;
                const int wo = wn / g.sw;
                if (wo >= g.Wo) continue;
                const int64_t q = (((int64_t)n * g.Ho + ho) * g.Wo + wo) * g.C + c0;
                float fy[VN], fd[VN];
                unsigned char ib[VN];
                unpack<T>(__ldg(reinterpret_cast<const uint4 *>(y + q)), fy);
                unpack<T>(__ldg(reinterpret_cast<const uint4 *>(dy + q)), fd);
                load_bytes<VN>(idx + q, ib);
#pragma unroll
                for (int e = 0; e < VN; ++e)
                    if (ib[e] == i * g.kw + j && fy[e] > 0.f) acc[e] += fd[e];
            }
        }
        const uint4 packed = pack<T>(acc);
        reinterpret_cast<uint4 *>(dz)[t] = packed;
        if (bias_sums || part) {         // sum what was actually stored (the rounded values), like a separate pass would
            float fr[VN];
            unpack<T>(packed, fr);
#pragma unroll
            for (int e = 0; e < VN; ++e) bsum[e] += fr[e];
        }
    }
    if (bias_sums || part) {             // only launched with blockDim % cv == 0: the channel vector is thread-invariant
        __shared__ float red[256][VN + 1];
        if (part) block_channel_partial<VN>(bsum, cv, part + (int64_t)blockIdx.x * g.C, red);
        else block_channel_sum<VN>(bsum, cv, bias_sums, red);
    }
}

// Non-overlapping windows (kernel == stride, no padding: the two big 2x2/2 pools of the CRNN stack): one thread per
// POOLED output vector reads y / dy / idx once and writes all kh*kw input positions of its window (dy at the arg-max
// if y > 0, zeros elsewhere) -- no div/mod per input pixel and no 4x re-read of the pooled tensors.
// Requires H % kh == 0 and W % kw == 0 so that every input pixel belongs to exactly one window.
template <typename T>
__global__ void __launch_bounds__(256)
bias_relu_pool_bwd_tiled_kernel(PoolGeo g, const T *__restrict__ dy, const T *__restrict__ y,
                                const unsigned char *__restrict__ idx, T *__restrict__ dz, double *__restrict__ bias_sums,
                                float *__restrict__ part) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = g.C / VN;
    const int64_t total = (int64_t)g.N * g.Ho * g.Wo * cv;
    float bsum[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) bsum[e] = 0.f;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int c0 = (int)(t % cv) * VN;
        const int64_t p = t / cv;
        const int wo = (int)(p % g.Wo);
        const int64_t r = p / g.Wo;
        const int ho = (int)(r % g.Ho);
        const int n = (int)(r / g.Ho);
        float fy[VN], fd[VN];
        unsigned char ib[VN];
        unpack<T>(__ldg(reinterpret_cast<const uint4 *>(y) + t), fy);
        unpack<T>(__ldg(reinterpret_cast<const uint4 *>(dy) + t), fd);
        load_bytes<VN>(idx + t * VN, ib);
#pragma unroll
        for (int e = 0; e < VN; ++e) {
            if (!(fy[e] > 0.f)) fd[e] = 0.f;        // ReLU' through the pooled value
            bsum[e] += to_f<T>(from_f<T>(fd[e]));
        }
        for (int i = 0; i < g.kh; ++i)
            for (int j = 0; j < g.kw; ++j) {
                float o[VN];
#pragma unroll
                for (int e = 0; e < VN; ++e) o[e] = (ib[e] == i * g.kw + j) ? fd[e] : 0.f;
                const int64_t q = (((int64_t)n * g.H + ho * g.kh + i) * g.W + wo * g.kw + j) * g.C + c0;
                __stcs(reinterpret_cast<uint4 *>(dz + q), pack<T>(o));
            }
    }
    if (bias_sums || part) {
        __shared__ float red[256][VN + 1];
        if (part) block_channel_partial<VN>(bsum, cv, part + (int64_t)blockIdx.x * g.C, red);
        else block_channel_sum<VN>(bsum, cv, bias_sums, red);
    }
}

// ---- row-organised 2x2-window variants (every pool of the CRNN stack: backbones/crnn.py:18-35) -------------------------
// One block walks output rows (n, ho); threads walk (wo, channel-vector) items with the channel vector fixed per thread
// (256 % cv == 0, cv a power of two), so there is no 64-bit div/mod per element, the bias vector sits in registers and
// all window loads of an item are issued before the first compare.
template <typename T, int KH, int KW>
__global__ void __launch_bounds__(256)
pool_fwd_rows_kernel(PoolGeo g, const T *__restrict__ x, const float *__restrict__ bias, T *__restrict__ y,
                     unsigned char *__restrict__ idx, int cv_shift) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = 1 << cv_shift;
    const int cvec = threadIdx.x & (cv - 1), wl = threadIdx.x >> cv_shift, WL = 256 >> cv_shift;
    float bb[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) bb[e] = bias[cvec * VN + e];
    const uint4 *px = reinterpret_cast<const uint4 *>(x) + cvec;
    const int nrows = g.N * g.Ho;
    for (int row = blockIdx.x; row < nrows; row += gridDim.x) {
        const int n = row / g.Ho, ho = row - n * g.Ho;
        const int h0 = ho * g.sh - g.ph;
        for (int wo = wl; wo < g.Wo; wo += WL) {
            const int w0 = wo * g.sw - g.pw;
            uint4 v[KH * KW];
            bool ok[KH * KW];
#pragma unroll
            for (int i = 0; i < KH; ++i)
#pragma unroll
                for (int j = 0; j < KW; ++j) {
                    const int h = h0 + i, w = w0 + j;
                    ok[i * KW + j] = h >= 0 && h < g.H && w >= 0 && w < g.W;
                    v[i * KW + j] = make_uint4(0, 0, 0, 0);
                    if (ok[i * KW + j]) v[i * KW + j] = __ldg(px + ((int64_t)(n * g.H + h) * g.W + w) * cv);
                }
            float best[VN];
            int bi[VN];
#pragma unroll
            for (int e = 0; e < VN; ++e) { best[e] = -INFINITY; bi[e] = 0; }
#pragma unroll
            for (int k = 0; k < KH * KW; ++k) {
                if (!ok[k]) continue;
                float f[VN];
                unpack<T>(v[k], f);
#pragma unroll
                for (int e = 0; e < VN; ++e) {
                    const float a = to_f<T>(from_f<T>(fmaxf(f[e] + bb[e], 0.f)));
                    if (a > best[e]) { best[e] = a; bi[e] = k; }
                }
            }
            const int64_t t = ((int64_t)row * g.Wo + wo) * cv + cvec;
            reinterpret_cast<uint4 *>(y)[t] = pack<T>(best);
            unsigned char ib[VN];
#pragma unroll
            for (int e = 0; e < VN; ++e) ib[e] = (unsigned char)bi[e];
            store_bytes<VN>(idx + t * VN, ib);
        }
    }
}

// backward, one block per INPUT row (n, h): every input pixel gathers from the <= KH*KW windows that contain it
template <typename T, int KH, int KW>
__global__ void __launch_bounds__(256)
pool_bwd_rows_kernel(PoolGeo g, const T *__restrict__ dy, const T *__restrict__ y, const unsigned char *__restrict__ idx,
                     T *__restrict__ dz, float *__restrict__ part, int cv_shift) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = 1 << cv_shift;
    const int cvec = threadIdx.x & (cv - 1), wl = threadIdx.x >> cv_shift, WL = 256 >> cv_shift;
    float bsum[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) bsum[e] = 0.f;
    const int nrows = g.N * g.H;
    for (int row = blockIdx.x; row < nrows; row += gridDim.x) {
        const int n = row / g.H, h = row - n * g.H;
        int hos[KH];                                             // pooled row reached through window offset i, or -1
#pragma unroll
        for (int i = 0; i < KH; ++i) {
            const int hn = h + g.ph - i;
            hos[i] = (hn >= 0 && hn % g.sh == 0 && hn / g.sh < g.Ho) ? hn / g.sh : -1;
        }
        for (int w = wl; w < g.W; w += WL) {
            uint4 vy[KH * KW], vd[KH * KW];
            unsigned char ib[KH * KW][VN];
            bool ok[KH * KW];
#pragma unroll
            for (int i = 0; i < KH; ++i)
#pragma unroll
                for (int j = 0; j < KW; ++j) {
                    const int k = i * KW + j;
                    const int wn = w + g.pw - j;
                    const int wo = wn / g.sw;
                    ok[k] = hos[i] >= 0 && wn >= 0 && wn % g.sw == 0 && wo < g.Wo;
                    if (ok[k]) {
                        const int64_t q = ((int64_t)(n * g.Ho + hos[i]) * g.Wo + wo) * cv + cvec;
                        vy[k] = __ldg(reinterpret_cast<const uint4 *>(y) + q);
                        vd[k] = __ldg(reinterpret_cast<const uint4 *>(dy) + q);
                        load_bytes<VN>(idx + q * VN, ib[k]);
                    }
                }
            float acc[VN];
#pragma unroll
            for (int e = 0; e < VN; ++e) acc[e] = 0.f;
#pragma unroll
            for (int k = 0; k < KH * KW; ++k) {
                if (!ok[k]) continue;
                float fy[VN], fd[VN];
                unpack<T>(vy[k], fy);
                unpack<T>(vd[k], fd);
#pragma unroll
                for (int e = 0; e < VN; ++e)
                    if (ib[k][e] == k && fy[e] > 0.f) acc[e] += fd[e];
            }
            const uint4 packed = pack<T>(acc);
            __stcs(reinterpret_cast<uint4 *>(dz) + ((int64_t)row * g.W + w) * cv + cvec, packed);
            if (part) {
                float fr[VN];
                unpack<T>(packed, fr);
#pragma unroll
                for (int e = 0; e < VN; ++e) bsum[e] += fr[e];
            }
        }
    }
    if (part) {
        __shared__ float red[256][VN + 1];
        block_channel_partial<VN>(bsum, cv, part + (int64_t)blockIdx.x * g.C, red);
    }
}

// backward for windows that tile the height exactly (kh == sh == 2, no vertical padding, H even) but may overlap along
// the width (the (2,1)-stride pools of the CRNN stack): one block per POOLED row (n, ho); a thread owns input column w
// for BOTH input rows 2*ho and 2*ho+1, so each contributing window (y, dy, arg-max) is loaded once instead of twice.
template <typename T, int KW>
__global__ void __launch_bounds__(256)
pool_bwd_hpair_rows_kernel(PoolGeo g, const T *__restrict__ dy, const T *__restrict__ y, const unsigned char *__restrict__ idx,
                           T *__restrict__ dz, float *__restrict__ part, int cv_shift) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = 1 << cv_shift;
    const int cvec = threadIdx.x & (cv - 1), wl = threadIdx.x >> cv_shift, WL = 256 >> cv_shift;
    float bsum[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) bsum[e] = 0.f;
    const int nrows = g.N * g.Ho;
    for (int row = blockIdx.x; row < nrows; row += gridDim.x) {
        const int n = row / g.Ho, ho = row - n * g.Ho;
        for (int w = wl; w < g.W; w += WL) {
            uint4 vy[KW], vd[KW];
            unsigned char ib[KW][VN];
            bool ok[KW];
#pragma unroll
            for (int j = 0; j < KW; ++j) {
                const int wn = w + g.pw - j;
                const int wo = wn / g.sw;
                ok[j] = wn >= 0 && wn % g.sw == 0 && wo < g.Wo;
                if (ok[j]) {
                    const int64_t q = ((int64_t)row * g.Wo + wo) * cv + cvec;
                    vy[j] = __ldg(reinterpret_cast<const uint4 *>(y) + q);
                    vd[j] = __ldg(reinterpret_cast<const uint4 *>(dy) + q);
                    load_bytes<VN>(idx + q * VN, ib[j]);
                }
            }
            float acc0[VN], acc1[VN];
#pragma unroll
            for (int e = 0; e < VN; ++e) acc0[e] = acc1[e] = 0.f;
#pragma unroll
            for (int j = 0; j < KW; ++j) {
                if (!ok[j]) continue;
                float fy[VN], fd[VN];
                unpack<T>(vy[j], fy);
                unpack<T>(vd[j], fd);
#pragma unroll
                for (int e = 0; e < VN; ++e) {
                    const float gsel = fy[e] > 0.f ? fd[e] : 0.f;
                    if (ib[j][e] == j) acc0[e] += gsel;              // arg-max in the upper row of the window (i = 0)
                    if (ib[j][e] == KW + j) acc1[e] += gsel;         // ... in the lower row (i = 1)
                }
            }
            const uint4 p0 = pack<T>(acc0), p1 = pack<T>(acc1);
            uint4 *o = reinterpret_cast<uint4 *>(dz) + ((int64_t)(n * g.H + 2 * ho) * g.W + w) * cv + cvec;
            __stcs(o, p0);
            __stcs(o + (int64_t)g.W * cv, p1);
            if (part) {
                float f0[VN], f1[VN];
                unpack<T>(p0, f0);
                unpack<T>(p1, f1);
#pragma unroll
                for (int e = 0; e < VN; ++e) bsum[e] += f0[e] + f1[e];
            }
        }
    }
    if (part) {
        __shared__ float red[256][VN + 1];
        block_channel_partial<VN>(bsum, cv, part + (int64_t)blockIdx.x * g.C, red);
    }
}

// backward for non-overlapping windows, one block per POOLED row (n, ho): read once, write the KH*KW input positions
template <typename T, int KH, int KW>
__global__ void __launch_bounds__(256)
pool_bwd_tiled_rows_kernel(PoolGeo g, const T *__restrict__ dy, const T *__restrict__ y,
                           const unsigned char *__restrict__ idx, T *__restrict__ dz, float *__restrict__ part, int cv_shift) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = 1 << cv_shift;
    const int cvec = threadIdx.x & (cv - 1), wl = threadIdx.x >> cv_shift, WL = 256 >> cv_shift;
    float bsum[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) bsum[e] = 0.f;
    const int nrows = g.N * g.Ho;
    for (int row = blockIdx.x; row < nrows; row += gridDim.x) {
        const int n = row / g.Ho, ho = row - n * g.Ho;
        for (int wo = wl; wo < g.Wo; wo += 2 * WL) {             // two pooled vectors in flight
            const int wo2 = wo + WL;
            const bool two = wo2 < g.Wo;
            const int64_t t = ((int64_t)row * g.Wo + wo) * cv + cvec, t2 = ((int64_t)row * g.Wo + wo2) * cv + cvec;
            uint4 ry[2], rd[2];
            unsigned char ib[2][VN];
            ry[0] = __ldg(reinterpret_cast<const uint4 *>(y) + t);
            rd[0] = __ldg(reinterpret_cast<const uint4 *>(dy) + t);
            load_bytes<VN>(idx + t * VN, ib[0]);
            if (two) {
                ry[1] = __ldg(reinterpret_cast<const uint4 *>(y) + t2);
                rd[1] = __ldg(reinterpret_cast<const uint4 *>(dy) + t2);
                load_bytes<VN>(idx + t2 * VN, ib[1]);
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                if (u == 1 && !two) break;
                float fy[VN], fd[VN];
                unpack<T>(ry[u], fy);
                unpack<T>(rd[u], fd);
#pragma unroll
                for (int e = 0; e < VN; ++e) {
                    if (!(fy[e] > 0.f)) fd[e] = 0.f;            // ReLU' through the pooled value
                    bsum[e] += to_f<T>(from_f<T>(fd[e]));
                }
                const int wcur = u ? wo2 : wo;
#pragma unroll
                for (int i = 0; i < KH; ++i)
#pragma unroll
                    for (int j = 0; j < KW; ++j) {
                        float o[VN];
#pragma unroll
                        for (int e = 0; e < VN; ++e) o[e] = (ib[u][e] == i * KW + j) ? fd[e] : 0.f;
                        const int64_t q = ((int64_t)(n * g.H + ho * KH + i) * g.W + wcur * KW + j) * cv + cvec;
                        __stcs(reinterpret_cast<uint4 *>(dz) + q, pack<T>(o));
                    }
            }
        }
    }
    if (part) {
        __shared__ float red[256][VN + 1];
        block_channel_partial<VN>(bsum, cv, part + (int64_t)blockIdx.x * g.C, red);
    }
}

inline int pow2_shift(int v) {      // log2(v) if v is a power of two, else -1
    if (v <= 0 || (v & (v - 1))) return -1;
    int sft = 0;
    while ((1 << sft) < v) ++sft;
    return sft;
}

// plain bias (+ optional ReLU) on [rows, C], and its backward mask
template <typename T>
__global__ void bias_act_kernel(const T *__restrict__ x, const float *__restrict__ bias, int64_t rows, int C, int relu,
                                T *__restrict__ y) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = C / VN;
    const int64_t total = rows * cv;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int c0 = (int)(t % cv) * VN;
        float f[VN];
        unpack<T>(__ldg(reinterpret_cast<const uint4 *>(x) + t), f);
#pragma unroll
        for (int e = 0; e < VN; ++e) {
            f[e] += bias[c0 + e];
            if (relu) f[e] = fmaxf(f[e], 0.f);
        }
        reinterpret_cast<uint4 *>(y)[t] = pack<T>(f);
    }
}

template <typename T>
__global__ void bias_act_scalar_kernel(const T *__restrict__ x, const float *__restrict__ bias, int64_t total, int C,
                                       int relu, T *__restrict__ y) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        float f = to_f<T>(x[t]) + bias[t % C];
        if (relu) f = fmaxf(f, 0.f);
        y[t] = from_f<T>(f);
    }
}

// ---------------------------------------------------------------- per-channel reductions over rows
// sums[0][c] += sum_r f(x[r,c] (+bias[c]));  sums[1][c] += sum_r g(...)   MODE 0: (x+b, (x+b)^2)   [BN statistics]
//                                                                          MODE 1: (dy, dy*xhat)      [BN backward]
//                                                                          MODE 2: (dy, -)            [bias gradient]
// xhat = (x + bias - mean) * invstd.  One CTA = 32 channel-vectors x 8 row lanes; double atomics at the end.
template <typename T, int MODE>
__global__ void __launch_bounds__(256)
col_reduce_kernel(const T *__restrict__ a, const T *__restrict__ b, const float *__restrict__ bias,
                  const float *__restrict__ mean, const float *__restrict__ invstd, int64_t rows, int C,
                  int64_t rows_per_cta, double *__restrict__ sums, float *__restrict__ part) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = C / VN;
    const int lane_c = threadIdx.x & 31, lane_r = threadIdx.x >> 5;   // 32 x 8
    const int v = blockIdx.x * 32 + lane_c;
    const int64_t r0 = (int64_t)blockIdx.y * rows_per_cta;
    const int64_t r1 = min(rows, r0 + rows_per_cta);
    float s0[VN], s1[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) s0[e] = s1[e] = 0.f;
    if (v < cv) {
        float bb[VN], mm[VN], is[VN];
#pragma unroll
        for (int e = 0; e < VN; ++e) {
            bb[e] = bias ? bias[v * VN + e] : 0.f;
            mm[e] = (MODE == 1) ? mean[v * VN + e] : 0.f;
            is[e] = (MODE == 1) ? invstd[v * VN + e] : 0.f;
        }
        constexpr int U = 4;             // rows in flight per thread
        for (int64_t r = r0 + lane_r; r < r1; r += 8 * U) {
            uint4 ra[U], rb[U];
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const int64_t rr = r + 8 * k;
                const bool ok = rr < r1;
                ra[k] = ok ? __ldg(reinterpret_cast<const uint4 *>(a + rr * C) + v) : make_uint4(0, 0, 0, 0);
                if (MODE == 1) rb[k] = ok ? __ldg(reinterpret_cast<const uint4 *>(b + rr * C) + v) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                if (r + 8 * k >= r1) break;
                float fa[VN];
                unpack<T>(ra[k], fa);
                if (MODE == 0) {
#pragma unroll
                    for (int e = 0; e < VN; ++e) { const float x = fa[e] + bb[e]; s0[e] += x; s1[e] += x * x; }
                } else if (MODE == 1) {
                    float fb[VN];
                    unpack<T>(rb[k], fb);
#pragma unroll
                    for (int e = 0; e < VN; ++e) { s0[e] += fa[e]; s1[e] += fa[e] * ((fb[e] + bb[e] - mm[e]) * is[e]); }
                } else {
#pragma unroll
                    for (int e = 0; e < VN; ++e) s0[e] += fa[e];
                }
            }
        }
    }
    __shared__ float red[2][8][32][VN + 1];
#pragma unroll
    for (int e = 0; e < VN; ++e) { red[0][lane_r][lane_c][e] = s0[e]; red[1][lane_r][lane_c][e] = s1[e]; }
    __syncthreads();
    if (lane_r == 0 && v < cv) {
#pragma unroll
        for (int e = 0; e < VN; ++e) {
            float t0 = 0.f, t1 = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) { t0 += red[0][k][lane_c][e]; t1 += red[1][k][lane_c][e]; }
            if (part) {                  // one row of [gridDim.y, 2C] per row block, added up by partials_finalize_kernel
                part[(int64_t)blockIdx.y * 2 * C + v * VN + e] = t0;
                part[(int64_t)blockIdx.y * 2 * C + C + v * VN + e] = (MODE != 2) ? t1 : 0.f;
            } else {
                atomicAdd(sums + v * VN + e, (double)t0);
                if (MODE != 2) atomicAdd(sums + C + v * VN + e, (double)t1);
            }
        }
    }
}

// BatchNorm finalize (one thread per channel): mean / invstd from the sums, running-stat update (momentum, unbiased
// variance for running_var like ATen), num_batches_tracked is bumped by the host.
__global__ void bn_finalize_kernel(const double *__restrict__ sums, int64_t rows, int C, float eps, float momentum,
                                   float *__restrict__ mean, float *__restrict__ invstd,
                                   float *__restrict__ running_mean, float *__restrict__ running_var) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const double m = sums[c] / (double)rows;
    double var = sums[C + c] / (double)rows - m * m;
    if (var < 0) var = 0;
    mean[c] = (float)m;
    invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
    if (running_mean) {
        const double unbiased = rows > 1 ? var * (double)rows / (double)(rows - 1) : var;
        running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * m);
        running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unbiased);
    }
}

// y = (x + bias - mean) * invstd * gamma + beta  ==  x * sc + sh  per channel
template <typename T>
__global__ void bn_apply_kernel(const T *__restrict__ x, const float *__restrict__ bias, const float *__restrict__ mean,
                                const float *__restrict__ invstd, const float *__restrict__ gamma,
                                const float *__restrict__ beta, int64_t rows, int C, T *__restrict__ y) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = C / VN;
    const int64_t total = rows * cv;
    float sc[VN], sh[VN];
    int c_cached = -1;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int c0 = (int)(t % cv) * VN;
        if (c0 != c_cached) {
#pragma unroll
            for (int e = 0; e < VN; ++e) {
                const int c = c0 + e;
                sc[e] = invstd[c] * gamma[c];
                sh[e] = ((bias ? bias[c] : 0.f) - mean[c]) * sc[e] + beta[c];
            }
            c_cached = c0;
        }
        float f[VN];
        unpack<T>(__ldg(reinterpret_cast<const uint4 *>(x) + t), f);
#pragma unroll
        for (int e = 0; e < VN; ++e) f[e] = f[e] * sc[e] + sh[e];
        reinterpret_cast<uint4 *>(y)[t] = pack<T>(f);
    }
}

// dx = gamma * invstd * (dy - sum_dy/rows - xhat * sum_dy_xhat/rows)
template <typename T>
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const T *__restrict__ dy, const T *__restrict__ x, const float *__restrict__ bias,
                    const float *__restrict__ mean, const float *__restrict__ invstd, const float *__restrict__ gamma,
                    const double *__restrict__ sums, int64_t rows, int C, T *__restrict__ dx,
                    double *__restrict__ bias_sums) {
    constexpr int VN = 16 / sizeof(T);
    const int cv = C / VN;
    const int64_t total = rows * cv;
    const float inv_rows = 1.f / (float)rows;
    float A[VN], k1[VN], k2[VN], shf[VN], is[VN], bsum[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) bsum[e] = 0.f;
    int c_cached = -1;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += 2 * stride) {
        const int c0 = (int)(t % cv) * VN;
        if (c0 != c_cached) {
#pragma unroll
            for (int e = 0; e < VN; ++e) {
                const int c = c0 + e;
                is[e] = invstd[c];
                A[e] = gamma[c] * is[e];
                k1[e] = (float)sums[c] * inv_rows;
                k2[e] = (float)sums[C + c] * inv_rows;
                shf[e] = (bias ? bias[c] : 0.f) - mean[c];
            }
            c_cached = c0;
        }
        // two independent vectors in flight per thread (the second shares the channel vector when cv | stride)
        const int64_t t2 = t + stride;
        const bool two = t2 < total && ((int)(t2 % cv) * VN == c0);
        uint4 rd = __ldg(reinterpret_cast<const uint4 *>(dy) + t), rx = __ldg(reinterpret_cast<const uint4 *>(x) + t);
        uint4 rd2 = rd, rx2 = rx;
        if (two) { rd2 = __ldg(reinterpret_cast<const uint4 *>(dy) + t2); rx2 = __ldg(reinterpret_cast<const uint4 *>(x) + t2); }
        float fd[VN], fx[VN];
        unpack<T>(rd, fd);
        unpack<T>(rx, fx);
#pragma unroll
        for (int e = 0; e < VN; ++e) fd[e] = A[e] * (fd[e] - k1[e] - (fx[e] + shf[e]) * is[e] * k2[e]);
        uint4 packed = pack<T>(fd);
        reinterpret_cast<uint4 *>(dx)[t] = packed;
        if (bias_sums) {
            float fr[VN];
            unpack<T>(packed, fr);
#pragma unroll
            for (int e = 0; e < VN; ++e) bsum[e] += fr[e];
        }
        if (two) {
            unpack<T>(rd2, fd);
            unpack<T>(rx2, fx);
#pragma unroll
            for (int e = 0; e < VN; ++e) fd[e] = A[e] * (fd[e] - k1[e] - (fx[e] + shf[e]) * is[e] * k2[e]);
            packed = pack<T>(fd);
            reinterpret_cast<uint4 *>(dx)[t2] = packed;
            if (bias_sums) {
                float fr[VN];
                unpack<T>(packed, fr);
#pragma unroll
                for (int e = 0; e < VN; ++e) bsum[e] += fr[e];
            }
        } else if (t2 < total) {
            // channel vector differs (cv does not divide the stride): handle it in the plain way
            const int c2 = (int)(t2 % cv) * VN;
            float gd[VN], gx[VN];
            unpack<T>(__ldg(reinterpret_cast<const uint4 *>(dy) + t2), gd);
            unpack<T>(__ldg(reinterpret_cast<const uint4 *>(x) + t2), gx);
#pragma unroll
            for (int e = 0; e < VN; ++e) {
                const int c = c2 + e;
                const float isv = invstd[c];
                gd[e] = gamma[c] * isv * (gd[e] - (float)sums[c] * inv_rows -
                                          (gx[e] + (bias ? bias[c] : 0.f) - mean[c]) * isv * (float)sums[C + c] * inv_rows);
            }
            reinterpret_cast<uint4 *>(dx)[t2] = pack<T>(gd);
        }
    }
    if (bias_sums) {
        __shared__ float red[256][VN + 1];
        block_channel_sum<VN>(bsum, cv, bias_sums, red);
    }
}

// Row-tiled variants of the two BatchNorm streaming kernels for 256 % (C / VN) == 0: a thread keeps ONE channel vector
// (coefficients live in registers, no per-element index arithmetic), a block owns a contiguous range of rows and keeps
// U rows per thread in flight.  Grid = one resident wave.
template <typename T>
__global__ void __launch_bounds__(256, 2)
bn_bwd_apply_rows_kernel(const T *__restrict__ dy, const T *__restrict__ x, const float *__restrict__ bias,
                         const float *__restrict__ mean, const float *__restrict__ invstd, const float *__restrict__ gamma,
                         const double *__restrict__ sums, int64_t rows, int C, int64_t rows_per_cta, T *__restrict__ dx,
                         float *__restrict__ part) {
    constexpr int VN = 16 / sizeof(T);
    constexpr int U = 4;
    const int cv = C / VN;
    const int cvec = threadIdx.x % cv, rl = threadIdx.x / cv, RL = 256 / cv;
    const float inv_rows = 1.f / (float)rows;
    float A[VN], k1[VN], t1[VN], shf[VN], bsum[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) {
        const int c = cvec * VN + e;
        const float is = invstd[c];
        A[e] = gamma[c] * is;
        k1[e] = (float)sums[c] * inv_rows;
        t1[e] = is * ((float)sums[C + c] * inv_rows);
        shf[e] = (bias ? bias[c] : 0.f) - mean[c];
        bsum[e] = 0.f;
    }
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
    const uint4 *pd = reinterpret_cast<const uint4 *>(dy) + cvec;
    const uint4 *px = reinterpret_cast<const uint4 *>(x) + cvec;
    uint4 *po = reinterpret_cast<uint4 *>(dx) + cvec;
    for (int64_t r = r0 + rl; r < r1; r += (int64_t)U * RL) {
        uint4 rd[U], rx[U];
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int64_t rr = r + (int64_t)k * RL;
            if (rr < r1) { rd[k] = __ldg(pd + rr * cv); rx[k] = __ldg(px + rr * cv); }
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int64_t rr = r + (int64_t)k * RL;
            if (rr >= r1) break;
            float fd[VN], fx[VN];
            unpack<T>(rd[k], fd);
            unpack<T>(rx[k], fx);
#pragma unroll
            for (int e = 0; e < VN; ++e) fd[e] = A[e] * (fd[e] - k1[e] - (fx[e] + shf[e]) * t1[e]);
            const uint4 packed = pack<T>(fd);
            __stcs(po + rr * cv, packed);
            if (part) {
                float fr[VN];
                unpack<T>(packed, fr);
#pragma unroll
                for (int e = 0; e < VN; ++e) bsum[e] += fr[e];
            }
        }
    }
    if (part) {
        __shared__ float red[256][VN + 1];
        block_channel_partial<VN>(bsum, cv, part + (int64_t)blockIdx.x * C, red);
    }
}

template <typename T>
__global__ void __launch_bounds__(256, 2)
bn_apply_rows_kernel(const T *__restrict__ x, const float *__restrict__ bias, const float *__restrict__ mean,
                     const float *__restrict__ invstd, const float *__restrict__ gamma, const float *__restrict__ beta,
                     int64_t rows, int C, int64_t rows_per_cta, T *__restrict__ y) {
    constexpr int VN = 16 / sizeof(T);
    constexpr int U = 4;
    const int cv = C / VN;
    const int cvec = threadIdx.x % cv, rl = threadIdx.x / cv, RL = 256 / cv;
    float sc[VN], sh[VN];
#pragma unroll
    for (int e = 0; e < VN; ++e) {
        const int c = cvec * VN + e;
        sc[e] = invstd[c] * gamma[c];
        sh[e] = ((bias ? bias[c] : 0.f) - mean[c]) * sc[e] + beta[c];
    }
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta, r1 = min(rows, r0 + rows_per_cta);
    const uint4 *px = reinterpret_cast<const uint4 *>(x) + cvec;
    uint4 *po = reinterpret_cast<uint4 *>(y) + cvec;
    for (int64_t r = r0 + rl; r < r1; r += (int64_t)U * RL) {
        uint4 rx[U];
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int64_t rr = r + (int64_t)k * RL;
            if (rr < r1) rx[k] = __ldg(px + rr * cv);
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int64_t rr = r + (int64_t)k * RL;
            if (rr >= r1) break;
            float f[VN];
            unpack<T>(rx[k], f);
#pragma unroll
            for (int e = 0; e < VN; ++e) f[e] = f[e] * sc[e] + sh[e];
            po[rr * cv] = pack<T>(f);
        }
    }
}

// rows per block for a one-wave grid of `per_sm` blocks per SM, rounded to the row step of the row-tiled kernels
inline int64_t rows_per_block(int64_t rows, int row_step, int per_sm, int *grid) {
    int64_t rpc = ceil_div(rows, (int64_t)mr::sm_count() * per_sm);
    rpc = ceil_div(rpc, (int64_t)row_step) * row_step;
    *grid = (int)ceil_div(rows, rpc);
    return rpc;
}

__global__ void sums_to_float_kernel(const double *__restrict__ s, int n, float scale, float *__restrict__ out, int accumulate) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (accumulate ? out[i] : 0.f) + scale * (float)s[i];
}

// ---------------------------------------------------------------- weight layout packs (one launch each instead of the
// permute / pad / flip / gather / contiguous / cast chains of the host code; the tensors are small and L2-resident)
// mode 0: conv weight [Cout,Cin,kh,kw] fp32 -> forward GEMM operand [Cout, Kp], column (i*kw + j)*Cp + c (zero padded)
// mode 1: -> input-gradient operand [Cin, kh*kw*Cout], column ((kh-1-i)*kw + (kw-1-j))*Cout + co  (flipped, transposed)
template <typename T>
__global__ void conv_weight_pack_kernel(const float *__restrict__ w, int Cout, int Cin, int kh, int kw, int Cp, int Kp,
                                        int mode, T *__restrict__ out) {
    const int64_t total = mode == 0 ? (int64_t)Cout * Kp : (int64_t)Cin * kh * kw * Cout;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        float v = 0.f;
        if (mode == 0) {
            const int co = (int)(t / Kp), col = (int)(t - (int64_t)co * Kp);
            if (col < kh * kw * Cp) {
                const int tap = col / Cp, c = col - tap * Cp;
                if (c < Cin) v = w[((int64_t)co * Cin + c) * kh * kw + tap];
            }
        } else {
            const int row = kh * kw * Cout;
            const int c = (int)(t / row), col = (int)(t - (int64_t)c * row);
            const int tapf = col / Cout, co = col - tapf * Cout;
            const int tap = kh * kw - 1 - tapf;                  // (kh-1-i')*kw + (kw-1-j')
            v = w[((int64_t)co * Cin + c) * kh * kw + tap];
        }
        out[t] = from_f<T>(v);
    }
}

// LSTM gate rows between the reference's gate-major order (row g*H + j) and the unit-major order of the wgmma kernels
// (row 4*j + g): out[r, :] = a[src(r), :] (+ b[src(r), :]);  inverse = 0: unit-major <- gate-major, 1: the way back.
template <typename T>
__global__ void gate_rows_permute_kernel(const float *__restrict__ a, const float *__restrict__ b, int H, int cols, int inverse,
                                         T *__restrict__ out) {
    const int64_t total = (int64_t)4 * H * cols;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(t / cols), k = (int)(t - (int64_t)r * cols);
        const int src = inverse ? ((r % H) * 4 + r / H) : ((r & 3) * H + (r >> 2));
        float v = a[(int64_t)src * cols + k];
        if (b) v += b[(int64_t)src * cols + k];
        out[t] = from_f<T>(v);
    }
}

// ---------------------------------------------------------------- LSTM cell (gate order i, f, g, o like ATen)
// One launch handles up to two directions (blockIdx.y): the forward and the reverse direction of a bidirectional
// layer advance in lock-step, so their cell updates share a launch.
// gates_pre [B, 4H] (T): x-projection + h_{t-1} W_hh^T already summed by the GEMMs; bias_ih + bias_hh added here.
// Writes the activated gates back in place (saved for backward), c_t [B,H] fp32, h_t [B,H] (T) into `h_out` (row
// stride ldh, so it lands directly in the [T, B, 2H] output of the bidirectional layer).
// bf16 mode uses MUFU.TANH (tanh.approx, ~2^-11 relative error, below bf16 resolution); fp32 mode keeps expf/tanhf
// so that the parity path stays within 1e-4 of the reference.
template <typename T> struct CellMath;
template <> struct CellMath<float> {
    static __device__ __forceinline__ float th(float x) { return tanhf(x); }
    static __device__ __forceinline__ float sg(float x) { return 1.f / (1.f + expf(-x)); }
};
template <> struct CellMath<bf16> {
    static __device__ __forceinline__ float th(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
    static __device__ __forceinline__ float sg(float x) { return fmaf(0.5f, th(0.5f * x), 0.5f); }
};

struct CellFwdDir { void *gates; const float *b_ih, *b_hh, *c_prev; float *c_out; void *h_out, *h_state; };
struct CellFwdArgs { CellFwdDir d[2]; int64_t ldh; int B, H; };

template <typename T>
__global__ void lstm_cell_fwd_kernel(CellFwdArgs a) {
    const CellFwdDir &q = a.d[blockIdx.y];
    T *gates = (T *)q.gates;
    T *h_out = (T *)q.h_out;
    T *h_state = (T *)q.h_state;
    const int H = a.H;
    const int64_t total = (int64_t)a.B * H;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(t / H), j = (int)(t - (int64_t)b * H);
        T *gp = gates + (int64_t)b * 4 * H;
        const float gi = to_f<T>(gp[j]) + q.b_ih[j] + q.b_hh[j];
        const float gf = to_f<T>(gp[H + j]) + q.b_ih[H + j] + q.b_hh[H + j];
        const float gg = to_f<T>(gp[2 * H + j]) + q.b_ih[2 * H + j] + q.b_hh[2 * H + j];
        const float go = to_f<T>(gp[3 * H + j]) + q.b_ih[3 * H + j] + q.b_hh[3 * H + j];
        const float i_ = CellMath<T>::sg(gi), f_ = CellMath<T>::sg(gf), g_ = CellMath<T>::th(gg), o_ = CellMath<T>::sg(go);
        const float c = f_ * (q.c_prev ? q.c_prev[t] : 0.f) + i_ * g_;
        const float h = o_ * CellMath<T>::th(c);
        gp[j] = from_f<T>(i_); gp[H + j] = from_f<T>(f_); gp[2 * H + j] = from_f<T>(g_); gp[3 * H + j] = from_f<T>(o_);
        q.c_out[t] = c;
        const T hv = from_f<T>(h);
        h_out[(int64_t)b * a.ldh + j] = hv;
        h_state[t] = hv;
    }
}

// dh_total = dh_out[t] (from the layer output gradient, row stride ldh) + dh_rec (from step t+1, may be NULL).
// Produces the pre-activation gate gradients dgates [B,4H] (T) and dc_prev (fp32, in place over dc).
struct CellBwdDir { const void *gates; const float *c, *c_prev; const void *dh_out, *dh_rec; float *dc; void *dgates; };
struct CellBwdArgs { CellBwdDir d[2]; int64_t ldh; int B, H; };

template <typename T>
__global__ void lstm_cell_bwd_kernel(CellBwdArgs a) {
    const CellBwdDir &q = a.d[blockIdx.y];
    const T *gates = (const T *)q.gates;
    const T *dh_out = (const T *)q.dh_out;
    const T *dh_rec = (const T *)q.dh_rec;
    T *dgates = (T *)q.dgates;
    const int H = a.H;
    const int64_t total = (int64_t)a.B * H;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(t / H), j = (int)(t - (int64_t)b * H);
        const T *gp = gates + (int64_t)b * 4 * H;
        const float i_ = to_f<T>(gp[j]), f_ = to_f<T>(gp[H + j]), g_ = to_f<T>(gp[2 * H + j]), o_ = to_f<T>(gp[3 * H + j]);
        const float dh = to_f<T>(dh_out[(int64_t)b * a.ldh + j]) + (dh_rec ? to_f<T>(dh_rec[t]) : 0.f);
        const float tc = CellMath<T>::th(q.c[t]);
        const float dct = q.dc[t] + dh * o_ * (1.f - tc * tc);
        const float cp = q.c_prev ? q.c_prev[t] : 0.f;
        T *dg = dgates + (int64_t)b * 4 * H;
        dg[j] = from_f<T>(dct * g_ * i_ * (1.f - i_));
        dg[H + j] = from_f<T>(dct * cp * f_ * (1.f - f_));
        dg[2 * H + j] = from_f<T>(dct * i_ * (1.f - g_ * g_));
        dg[3 * H + j] = from_f<T>(dh * tc * o_ * (1.f - o_));
        q.dc[t] = dct * f_;
    }
}

// ---------------------------------------------------------------- fused Adam over one flat fp32 buffer
// torch.optim.Adam semantics (no amsgrad, no weight decay): m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2;
// p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps).  Optionally refreshes a bf16 shadow copy of the parameters.
__global__ void adam_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m, float *__restrict__ v,
                            int64_t n, float lr, float b1, float b2, float eps, float bc1, float bc2_sqrt, float gscale,
                            bf16 *__restrict__ shadow) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float gi = g[i] * gscale;
        const float mi = b1 * m[i] + (1.f - b1) * gi;
        const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
        m[i] = mi; v[i] = vi;
        const float pi = p[i] - (lr / bc1) * mi / (sqrtf(vi) / bc2_sqrt + eps);
        p[i] = pi;
        if (shadow) shadow[i] = __float2bfloat16_rn(pi);
    }
}

// small-C fallback of the column sum (C not a multiple of the vector width, e.g. the 38 classes of the last Linear)
template <typename T>
__global__ void colsum_scalar_kernel(const T *__restrict__ a, int64_t rows, int C, double *__restrict__ sums) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float acc = 0.f;
        for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) acc += to_f<T>(a[r * C + c]);
        atomicAdd(sums + c, (double)acc);
    }
}

template <typename TI, typename TO>
__global__ void cast_kernel(const TI *__restrict__ x, int64_t n, TO *__restrict__ y) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        y[i] = from_f<TO>(to_f<TI>(x[i]));
}


// ---------------------------------------------------------------- greedy CTC decoding (SURVEY.md §8f row N1)
// structure/representers/ctc_representer.py:22-34 and ctc_representer2d.py:27-51: per column the arg-max class
// (2D: along the arg-max-height path of classify*mask), then the collapse rule: skip a column whose class equals the
// previous kept class OR is `unknown` (without updating `previous`); otherwise emit it unless it is blank, and
// remember it.  Output int32 [N, W], blank-padded.  One CTA per sample: threads = columns, thread 0 runs the scan.
__global__ void ctc_greedy_decode_kernel(const float *__restrict__ prob, const float *__restrict__ mask, int C, int H,
                                         int W, int64_t sN, int64_t sC, int64_t sH, int64_t sW, int64_t mN, int64_t mH,
                                         int64_t mW, int blank, int unknown, int *__restrict__ out) {
    extern __shared__ int pred[];
    const int n = blockIdx.x;
    const float *p = prob + (int64_t)n * sN;
    const float *m = mask ? mask + (int64_t)n * mN : nullptr;
    for (int w = threadIdx.x; w < W; w += blockDim.x) {
        int hbest = 0;
        if (H > 1 || m) {                       // arg-max over heights of max over classes of classify*mask
            float best = -INFINITY;
            for (int h = 0; h < H; ++h) {
                const float mv = m ? m[h * mH + w * mW] : 1.f;
                float cmax = -INFINITY;
                for (int c = 0; c < C; ++c) cmax = fmaxf(cmax, p[c * sC + h * sH + w * sW] * mv);
                if (cmax > best) { best = cmax; hbest = h; }
            }
        }
        const float mv = m ? m[hbest * mH + w * mW] : 1.f;
        float best = -INFINITY;
        int cbest = 0;
        for (int c = 0; c < C; ++c) {
            const float v = p[c * sC + hbest * sH + w * sW] * mv;
            if (v > best) { best = v; cbest = c; }          // first maximum wins
        }
        pred[w] = cbest;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int valid = 0, previous = blank;
        int *o = out + (int64_t)n * W;
        for (int w = 0; w < W; ++w) {
            const int c = pred[w];
            if (c == previous || c == unknown) continue;
            if (c != blank) o[valid++] = c;
            previous = c;
        }
        for (int w = valid; w < W; ++w) o[w] = blank;
    }
}

// sequence_recognition_representer.py:23-28: everything from the first blank on becomes blank (attention decoder output)
__global__ void blank_after_first_blank_kernel(int *__restrict__ pred, int N, int W, int blank) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    int *r = pred + (int64_t)n * W;
    bool seen = false;
    for (int w = 0; w < W; ++w) {
        seen = seen || (r[w] == blank);
        if (seen) r[w] = blank;
    }
}

#define DISPATCH(dtype, CALL)                                   \
    do { if ((dtype) == 0) { using T = float; CALL; }           \
         else if ((dtype) == 1) { using T = bf16; CALL; }       \
         else return MR_ERR_BAD_SHAPE; } while (0)

int vec_ok(int dtype, int C) { return C % (dtype == 0 ? 4 : 8) == 0; }

}  // namespace

extern "C" {

int mr_colsum(const void *a, int64_t rows, int C, int dtype, float *out, int accumulate, double *sums, void *stream);

int mr_nchw_to_nhwc(const float *x, int N, int C, int H, int W, int Cp, int dtype, void *y, void *stream) {
    if (N < 0 || C <= 0 || H <= 0 || W <= 0 || Cp < C) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!x || !y) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH(dtype, (nchw_to_nhwc_kernel<T><<<grid1d((int64_t)N * H * W, 256), 256, 0, st>>>(x, N, C, H * W, Cp, (T *)y)));
    return check_launch("nchw_to_nhwc_kernel");
}

int mr_nhwc_to_nchw(const void *x, int N, int C, int H, int W, int Cp, int dtype, float *y, void *stream) {
    if (N < 0 || C <= 0 || H <= 0 || W <= 0 || Cp < C) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!x || !y) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH(dtype, (nhwc_to_nchw_kernel<T><<<grid1d((int64_t)N * C * H * W, 256), 256, 0, st>>>((const T *)x, N, C, H * W, Cp, y)));
    return check_launch("nhwc_to_nchw_kernel");
}

static int conv_geo(ConvGeo &g, int N, int H, int W, int C, int kh, int kw, int ph, int pw, int Kp) {
    if (N < 0 || H <= 0 || W <= 0 || C <= 0 || kh <= 0 || kw <= 0 || ph < 0 || pw < 0) return MR_ERR_BAD_SHAPE;
    g.N = N; g.H = H; g.W = W; g.C = C; g.kh = kh; g.kw = kw; g.ph = ph; g.pw = pw;
    g.Ho = H + 2 * ph - kh + 1; g.Wo = W + 2 * pw - kw + 1; g.K = kh * kw * C; g.Kp = Kp;
    if (g.Ho <= 0 || g.Wo <= 0 || Kp < g.K) return MR_ERR_BAD_SHAPE;
    return MR_OK;
}

/* col [N*Ho*Wo, Kp] from NHWC x; stride-1 convolution geometry (all the CRNN stack uses, backbones/crnn.py:8-10). */
int mr_im2col_nhwc(const void *x, int N, int H, int W, int C, int kh, int kw, int ph, int pw, int Kp, int dtype,
                   void *col, void *stream) {
    ConvGeo g;
    int rc = conv_geo(g, N, H, W, C, kh, kw, ph, pw, Kp);
    if (rc) return rc;
    if (N == 0) return MR_OK;
    if (!x || !col) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t P = (int64_t)N * g.Ho * g.Wo;
    if (vec_ok(dtype, C) && vec_ok(dtype, Kp)) {
        const int vn = dtype == 0 ? 4 : 8;
        DISPATCH(dtype, (im2col_vec_kernel<T><<<grid1d(P * (Kp / vn), 256, 32), 256, 0, st>>>(g, (const T *)x, (T *)col)));
    } else {
        DISPATCH(dtype, (im2col_scalar_kernel<T><<<grid1d(P * Kp, 256, 32), 256, 0, st>>>(g, (const T *)x, (T *)col)));
    }
    return check_launch("im2col_kernel");
}

/* dx NHWC [N,H,W,C] from dcol [N*Ho*Wo, Kp]  (adjoint of mr_im2col_nhwc). */
int mr_col2im_nhwc(const void *dcol, int N, int H, int W, int C, int kh, int kw, int ph, int pw, int Kp, int dtype,
                   void *dx, void *stream) {
    ConvGeo g;
    int rc = conv_geo(g, N, H, W, C, kh, kw, ph, pw, Kp);
    if (rc) return rc;
    if (N == 0) return MR_OK;
    if (!dcol || !dx) return MR_ERR_NULL_POINTER;
    if (!vec_ok(dtype, C) || !vec_ok(dtype, Kp)) return MR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const int vn = dtype == 0 ? 4 : 8;
    DISPATCH(dtype, (col2im_vec_kernel<T><<<grid1d((int64_t)N * H * W * (C / vn), 256, 32), 256, 0, st>>>(g, (const T *)dcol, (T *)dx)));
    return check_launch("col2im_kernel");
}

static int pool_geo(PoolGeo &g, int N, int H, int W, int C, int kh, int kw, int sh, int sw, int ph, int pw) {
    if (N < 0 || H <= 0 || W <= 0 || C <= 0 || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || ph < 0 || pw < 0 || kh * kw > 255)
        return MR_ERR_BAD_SHAPE;
    g.N = N; g.H = H; g.W = W; g.C = C; g.kh = kh; g.kw = kw; g.sh = sh; g.sw = sw; g.ph = ph; g.pw = pw;
    g.Ho = (H + 2 * ph - kh) / sh + 1; g.Wo = (W + 2 * pw - kw) / sw + 1;   /* floor mode, nn.MaxPool2d default */
    if (g.Ho <= 0 || g.Wo <= 0) return MR_ERR_BAD_SHAPE;
    return MR_OK;
}

/* y = maxpool(relu(x + bias)), idx = arg-max inside the window (uint8). */
int mr_bias_relu_pool_fwd(const void *x, const float *bias, int N, int H, int W, int C, int kh, int kw, int sh, int sw,
                          int ph, int pw, int dtype, void *y, unsigned char *idx, void *stream) {
    PoolGeo g;
    int rc = pool_geo(g, N, H, W, C, kh, kw, sh, sw, ph, pw);
    if (rc) return rc;
    if (N == 0) return MR_OK;
    if (!x || !bias || !y || !idx) return MR_ERR_NULL_POINTER;
    if (!vec_ok(dtype, C)) return MR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const int vn = dtype == 0 ? 4 : 8;
    const int sft = pow2_shift(C / vn);
    if (kh == 2 && kw == 2 && sft >= 0 && sft <= 8 && (int64_t)N * H * W < ((int64_t)1 << 31)) {
        const int nblocks = (int)std::min<int64_t>((int64_t)N * g.Ho, mr::sm_count() * 16);
        DISPATCH(dtype, (pool_fwd_rows_kernel<T, 2, 2><<<nblocks, 256, 0, st>>>(g, (const T *)x, bias, (T *)y, idx, sft)));
        return check_launch("pool_fwd_rows_kernel");
    }
    DISPATCH(dtype, (bias_relu_pool_fwd_kernel<T><<<grid1d((int64_t)N * g.Ho * g.Wo * (C / vn), 256, 32), 256, 0, st>>>(g, (const T *)x, bias, (T *)y, idx)));
    return check_launch("bias_relu_pool_fwd_kernel");
}

int mr_bias_relu_pool_bwd(const void *dy, const void *y, const unsigned char *idx, int N, int H, int W, int C, int kh,
                          int kw, int sh, int sw, int ph, int pw, int dtype, void *dz, float *dbias, double *sums,
                          void *stream) {
    PoolGeo g;
    int rc = pool_geo(g, N, H, W, C, kh, kw, sh, sw, ph, pw);
    if (rc) return rc;
    if (N == 0) return MR_OK;
    if (!dy || !y || !idx || !dz) return MR_ERR_NULL_POINTER;
    if (!vec_ok(dtype, C)) return MR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const int vn = dtype == 0 ? 4 : 8;
    const bool fuse = dbias && sums && (256 % (C / vn) == 0);
    float *part = (fuse && C <= kMaxPartialCols) ? partials_scratch() : nullptr;
    if (fuse && !part) MR_CUDA_TRY(cudaMemsetAsync(sums, 0, sizeof(double) * C, st), "memset sums");
    const bool tiled = kh == sh && kw == sw && ph == 0 && pw == 0 && H % kh == 0 && W % kw == 0;
    const int per_sm = part ? 8 : 32;                /* the partial-sum scratch has one row per block */
    int nblocks;
    const int sft = pow2_shift(C / vn);
    if (kh == 2 && kw == 2 && sft >= 0 && sft <= 8 && (part || !dbias) && (int64_t)N * H * W < ((int64_t)1 << 31)) {
        if (tiled) {
            nblocks = (int)std::min<int64_t>((int64_t)N * g.Ho, kMaxPartialBlocks);
            DISPATCH(dtype, (pool_bwd_tiled_rows_kernel<T, 2, 2><<<nblocks, 256, 0, st>>>(g, (const T *)dy, (const T *)y, idx, (T *)dz, part, sft)));
        } else if (sh == 2 && ph == 0 && H % 2 == 0 && g.Ho * 2 == H) {
            nblocks = (int)std::min<int64_t>((int64_t)N * g.Ho, kMaxPartialBlocks);
            DISPATCH(dtype, (pool_bwd_hpair_rows_kernel<T, 2><<<nblocks, 256, 0, st>>>(g, (const T *)dy, (const T *)y, idx, (T *)dz, part, sft)));
        } else {
            nblocks = (int)std::min<int64_t>((int64_t)N * H, kMaxPartialBlocks);
            DISPATCH(dtype, (pool_bwd_rows_kernel<T, 2, 2><<<nblocks, 256, 0, st>>>(g, (const T *)dy, (const T *)y, idx, (T *)dz, part, sft)));
        }
    } else if (tiled) {
        nblocks = grid1d((int64_t)N * g.Ho * g.Wo * (C / vn), 256, per_sm);
        DISPATCH(dtype, (bias_relu_pool_bwd_tiled_kernel<T><<<nblocks, 256, 0, st>>>(g, (const T *)dy, (const T *)y, idx, (T *)dz, (fuse && !part) ? sums : nullptr, part)));
    } else {
        nblocks = grid1d((int64_t)N * H * W * (C / vn), 256, per_sm);
        DISPATCH(dtype, (bias_relu_pool_bwd_kernel<T><<<nblocks, 256, 0, st>>>(g, (const T *)dy, (const T *)y, idx, (T *)dz, (fuse && !part) ? sums : nullptr, part)));
    }
    if (part) {
        rc = check_launch("bias_relu_pool_bwd_kernel");
        if (rc) return rc;
        partials_finalize_kernel<<<(int)ceil_div(C, 32), dim3(32, 32), 0, st>>>(part, nblocks, C, sums);
    }
    rc = check_launch("bias_relu_pool_bwd_kernel");
    if (rc || !dbias) return rc;
    if (!fuse) return mr_colsum(dz, (int64_t)N * H * W, C, dtype, dbias, 0, sums, stream);
    sums_to_float_kernel<<<(int)ceil_div(C, 128), 128, 0, st>>>(sums, C, 1.f, dbias, 0);
    return check_launch("sums_to_float_kernel");
}

int mr_bias_act(const void *x, const float *bias, int64_t rows, int C, int relu, int dtype, void *y, void *stream) {
    if (rows < 0 || C <= 0) return MR_ERR_BAD_SHAPE;
    if (rows == 0) return MR_OK;
    if (!x || !bias || !y) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    if (!vec_ok(dtype, C)) {
        DISPATCH(dtype, (bias_act_scalar_kernel<T><<<grid1d(rows * C, 256, 32), 256, 0, st>>>((const T *)x, bias, rows * C, C, relu, (T *)y)));
        return check_launch("bias_act_scalar_kernel");
    }
    const int vn = dtype == 0 ? 4 : 8;
    DISPATCH(dtype, (bias_act_kernel<T><<<grid1d(rows * (C / vn), 256, 32), 256, 0, st>>>((const T *)x, bias, rows, C, relu, (T *)y)));
    return check_launch("bias_act_kernel");
}

static int launch_reduce(int mode, int dtype, const void *a, const void *b, const float *bias, const float *mean,
                         const float *invstd, int64_t rows, int C, double *sums, cudaStream_t st) {
    if (!vec_ok(dtype, C)) return MR_ERR_UNSUPPORTED;
    const int vn = dtype == 0 ? 4 : 8;
    const int cv = C / vn;
    const int gx = (int)ceil_div(cv, 32);
    int64_t gy = (mr::sm_count() * 8) / gx;
    if (gy < 1) gy = 1;
    int64_t rpc = ceil_div(rows, gy);
    if (rpc < 64) rpc = 64;
    gy = ceil_div(rows, rpc);
    float *part = (gy <= kMaxPartialBlocks && 2 * C <= kMaxPartialCols) ? partials_scratch() : nullptr;
    if (!part) MR_CUDA_TRY(cudaMemsetAsync(sums, 0, sizeof(double) * 2 * C, st), "memset sums");
    dim3 grid(gx, (unsigned)gy);
#define RL(MODEV) DISPATCH(dtype, (col_reduce_kernel<T, MODEV><<<grid, 256, 0, st>>>((const T *)a, (const T *)b, bias, mean, invstd, rows, C, rpc, sums, part)))
    if (mode == 0) RL(0); else if (mode == 1) RL(1); else RL(2);
#undef RL
    if (part) {
        int rc = check_launch("col_reduce_kernel");
        if (rc) return rc;
        partials_finalize_kernel<<<(int)ceil_div(2 * C, 32), dim3(32, 32), 0, st>>>(part, (int)gy, 2 * C, sums);
        return check_launch("partials_finalize_kernel");
    }
    return check_launch("col_reduce_kernel");
}

/* Training-mode BatchNorm over [rows, C] of (x + bias): batch statistics, running-stat update, normalisation.
 * `sums` is a caller-provided scratch of 2*C doubles.  mean / invstd [C] are saved for the backward. */
int mr_bn_train_fwd(const void *x, const float *bias, const float *gamma, const float *beta, float *running_mean,
                    float *running_var, float momentum, float eps, int64_t rows, int C, int dtype, void *y, float *mean,
                    float *invstd, double *sums, void *stream) {
    if (rows <= 0 || C <= 0) return MR_ERR_BAD_SHAPE;
    if (!x || !gamma || !beta || !y || !mean || !invstd || !sums) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = launch_reduce(0, dtype, x, nullptr, bias, nullptr, nullptr, rows, C, sums, st);
    if (rc) return rc;
    bn_finalize_kernel<<<(int)ceil_div(C, 128), 128, 0, st>>>(sums, rows, C, eps, momentum, mean, invstd, running_mean, running_var);
    rc = check_launch("bn_finalize_kernel");
    if (rc) return rc;
    const int vn = dtype == 0 ? 4 : 8;
    if (256 % (C / vn) == 0) {
        int grid;
        const int64_t rpc = rows_per_block(rows, 4 * (256 / (C / vn)), 2, &grid);
        DISPATCH(dtype, (bn_apply_rows_kernel<T><<<grid, 256, 0, st>>>((const T *)x, bias, mean, invstd, gamma, beta, rows, C, rpc, (T *)y)));
    } else {
        DISPATCH(dtype, (bn_apply_kernel<T><<<grid1d(rows * (C / vn), 256, 32), 256, 0, st>>>((const T *)x, bias, mean, invstd, gamma, beta, rows, C, (T *)y)));
    }
    return check_launch("bn_apply_kernel");
}

/* Inference BatchNorm with given statistics (eval branch): y = (x + bias - mean) * invstd * gamma + beta. */
int mr_bn_apply(const void *x, const float *bias, const float *mean, const float *invstd, const float *gamma,
                const float *beta, int64_t rows, int C, int dtype, void *y, void *stream) {
    if (rows < 0 || C <= 0) return MR_ERR_BAD_SHAPE;
    if (rows == 0) return MR_OK;
    if (!x || !mean || !invstd || !gamma || !beta || !y) return MR_ERR_NULL_POINTER;
    if (!vec_ok(dtype, C)) return MR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const int vn = dtype == 0 ? 4 : 8;
    if (256 % (C / vn) == 0) {
        int grid;
        const int64_t rpc = rows_per_block(rows, 4 * (256 / (C / vn)), 2, &grid);
        DISPATCH(dtype, (bn_apply_rows_kernel<T><<<grid, 256, 0, st>>>((const T *)x, bias, mean, invstd, gamma, beta, rows, C, rpc, (T *)y)));
    } else {
        DISPATCH(dtype, (bn_apply_kernel<T><<<grid1d(rows * (C / vn), 256, 32), 256, 0, st>>>((const T *)x, bias, mean, invstd, gamma, beta, rows, C, (T *)y)));
    }
    return check_launch("bn_apply_kernel");
}

/* BatchNorm backward: dx (gradient w.r.t. x + bias), dgamma, dbeta (fp32, assigned). */
int mr_bn_train_bwd(const void *dy, const void *x, const float *bias, const float *mean, const float *invstd,
                    const float *gamma, int64_t rows, int C, int dtype, void *dx, float *dgamma, float *dbeta,
                    float *dbias, double *sums, void *stream) {
    if (rows <= 0 || C <= 0) return MR_ERR_BAD_SHAPE;
    if (!dy || !x || !mean || !invstd || !gamma || !dx || !dgamma || !dbeta || !sums) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = launch_reduce(1, dtype, dy, x, bias, mean, invstd, rows, C, sums, st);
    if (rc) return rc;
    sums_to_float_kernel<<<(int)ceil_div(C, 128), 128, 0, st>>>(sums, C, 1.f, dbeta, 0);
    sums_to_float_kernel<<<(int)ceil_div(C, 128), 128, 0, st>>>(sums + C, C, 1.f, dgamma, 0);
    rc = check_launch("sums_to_float_kernel");
    if (rc) return rc;
    const int vn = dtype == 0 ? 4 : 8;
    /* `sums` holds 2*C doubles of statistics + C more for the fused conv-bias gradient (sum of dx). */
    const int cv = C / vn;
    const bool fuse = dbias && vec_ok(dtype, C) && (256 % cv == 0);
    if (vec_ok(dtype, C) && 256 % cv == 0) {
        int grid;
        const int64_t rpc = rows_per_block(rows, 4 * (256 / cv), 2, &grid);
        float *part = (fuse && C <= kMaxPartialCols) ? partials_scratch() : nullptr;
        DISPATCH(dtype, (bn_bwd_apply_rows_kernel<T><<<grid, 256, 0, st>>>((const T *)dy, (const T *)x, bias, mean, invstd, gamma, sums, rows, C, rpc, (T *)dx, part)));
        rc = check_launch("bn_bwd_apply_rows_kernel");
        if (rc || !dbias) return rc;
        if (!part) return mr_colsum(dx, rows, C, dtype, dbias, 0, sums, stream);
        partials_finalize_kernel<<<(int)ceil_div(C, 32), dim3(32, 32), 0, st>>>(part, grid, C, sums + 2 * C);
        sums_to_float_kernel<<<(int)ceil_div(C, 128), 128, 0, st>>>(sums + 2 * C, C, 1.f, dbias, 0);
        return check_launch("sums_to_float_kernel");
    }
    if (fuse) MR_CUDA_TRY(cudaMemsetAsync(sums + 2 * C, 0, sizeof(double) * C, st), "memset sums");
    DISPATCH(dtype, (bn_bwd_apply_kernel<T><<<grid1d(rows * (C / vn), 256, 32), 256, 0, st>>>((const T *)dy, (const T *)x, bias, mean, invstd, gamma, sums, rows, C, (T *)dx, fuse ? sums + 2 * C : nullptr)));
    rc = check_launch("bn_bwd_apply_kernel");
    if (rc || !dbias) return rc;
    if (!fuse) return mr_colsum(dx, rows, C, dtype, dbias, 0, sums, stream);
    sums_to_float_kernel<<<(int)ceil_div(C, 128), 128, 0, st>>>(sums + 2 * C, C, 1.f, dbias, 0);
    return check_launch("sums_to_float_kernel");
}

/* out[c] (= or +=) sum_r a[r, c]  — bias gradients. */
int mr_colsum(const void *a, int64_t rows, int C, int dtype, float *out, int accumulate, double *sums, void *stream) {
    if (rows < 0 || C <= 0) return MR_ERR_BAD_SHAPE;
    if (!a || !out || !sums) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    if (!vec_ok(dtype, C)) {
        MR_CUDA_TRY(cudaMemsetAsync(sums, 0, sizeof(double) * C, st), "memset sums");
        DISPATCH(dtype, (colsum_scalar_kernel<T><<<grid1d(rows, 256, 4), 256, 0, st>>>((const T *)a, rows, C, sums)));
        int rc0 = check_launch("colsum_scalar_kernel");
        if (rc0) return rc0;
        sums_to_float_kernel<<<(int)ceil_div(C, 128), 128, 0, st>>>(sums, C, 1.f, out, accumulate);
        return check_launch("sums_to_float_kernel");
    }
    int rc = launch_reduce(2, dtype, a, nullptr, nullptr, nullptr, nullptr, rows, C, sums, st);
    if (rc) return rc;
    sums_to_float_kernel<<<(int)ceil_div(C, 128), 128, 0, st>>>(sums, C, 1.f, out, accumulate);
    return check_launch("sums_to_float_kernel");
}

/* ndir = 1 or 2 directions per launch; the per-direction pointers are arrays of length ndir. */
int mr_lstm_cell_fwd(void *const *gates, const float *const *b_ih, const float *const *b_hh, const float *const *c_prev,
                     float *const *c_out, void *const *h_out, int64_t ldh, void *const *h_state, int ndir, int B, int H,
                     int dtype, void *stream) {
    if (B <= 0 || H <= 0 || ndir < 1 || ndir > 2) return MR_ERR_BAD_SHAPE;
    if (!gates || !b_ih || !b_hh || !c_prev || !c_out || !h_out || !h_state) return MR_ERR_NULL_POINTER;
    CellFwdArgs a;
    a.ldh = ldh; a.B = B; a.H = H;
    for (int d = 0; d < ndir; ++d) {
        if (!gates[d] || !b_ih[d] || !b_hh[d] || !c_out[d] || !h_out[d] || !h_state[d]) return MR_ERR_NULL_POINTER;
        a.d[d].gates = gates[d]; a.d[d].b_ih = b_ih[d]; a.d[d].b_hh = b_hh[d]; a.d[d].c_prev = c_prev[d];
        a.d[d].c_out = c_out[d]; a.d[d].h_out = h_out[d]; a.d[d].h_state = h_state[d];
    }
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(grid1d((int64_t)B * H, 256), ndir);
    DISPATCH(dtype, (lstm_cell_fwd_kernel<T><<<grid, 256, 0, st>>>(a)));
    return check_launch("lstm_cell_fwd_kernel");
}

int mr_lstm_cell_bwd(const void *const *gates, const float *const *c, const float *const *c_prev,
                     const void *const *dh_out, int64_t ldh, const void *const *dh_rec, float *const *dc,
                     void *const *dgates, int ndir, int B, int H, int dtype, void *stream) {
    if (B <= 0 || H <= 0 || ndir < 1 || ndir > 2) return MR_ERR_BAD_SHAPE;
    if (!gates || !c || !c_prev || !dh_out || !dh_rec || !dc || !dgates) return MR_ERR_NULL_POINTER;
    CellBwdArgs a;
    a.ldh = ldh; a.B = B; a.H = H;
    for (int d = 0; d < ndir; ++d) {
        if (!gates[d] || !c[d] || !dh_out[d] || !dc[d] || !dgates[d]) return MR_ERR_NULL_POINTER;
        a.d[d].gates = gates[d]; a.d[d].c = c[d]; a.d[d].c_prev = c_prev[d]; a.d[d].dh_out = dh_out[d];
        a.d[d].dh_rec = dh_rec[d]; a.d[d].dc = dc[d]; a.d[d].dgates = dgates[d];
    }
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(grid1d((int64_t)B * H, 256), ndir);
    DISPATCH(dtype, (lstm_cell_bwd_kernel<T><<<grid, 256, 0, st>>>(a)));
    return check_launch("lstm_cell_bwd_kernel");
}

int mr_adam_step(float *p, const float *g, float *m, float *v, int64_t n, float lr, float beta1, float beta2, float eps,
                 int64_t step, float grad_scale, void *bf16_shadow, void *stream) {
    if (n < 0 || step < 1) return MR_ERR_BAD_SHAPE;
    if (n == 0) return MR_OK;
    if (!p || !g || !m || !v) return MR_ERR_NULL_POINTER;
    const float bc1 = 1.f - powf(beta1, (float)step);
    const float bc2s = sqrtf(1.f - powf(beta2, (float)step));
    adam_kernel<<<grid1d(n, 256), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, n, lr, beta1, beta2, eps, bc1, bc2s, grad_scale, (bf16 *)bf16_shadow);
    return check_launch("adam_kernel");
}

int mr_cast(const void *x, int src_dtype, int64_t n, int dst_dtype, void *y, void *stream) {
    if (n < 0) return MR_ERR_BAD_SHAPE;
    if (n == 0) return MR_OK;
    if (!x || !y) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    const int g = grid1d(n, 256);
    if (src_dtype == 0 && dst_dtype == 1) cast_kernel<float, bf16><<<g, 256, 0, st>>>((const float *)x, n, (bf16 *)y);
    else if (src_dtype == 1 && dst_dtype == 0) cast_kernel<bf16, float><<<g, 256, 0, st>>>((const bf16 *)x, n, (float *)y);
    else if (src_dtype == 0 && dst_dtype == 0) cast_kernel<float, float><<<g, 256, 0, st>>>((const float *)x, n, (float *)y);
    else if (src_dtype == 1 && dst_dtype == 1) cast_kernel<bf16, bf16><<<g, 256, 0, st>>>((const bf16 *)x, n, (bf16 *)y);
    else return MR_ERR_BAD_SHAPE;
    return check_launch("cast_kernel");
}

/* Greedy CTC decoding to label indices (bit-exact integer output).  prob: class scores with element strides
 * (sN, sC, sH, sW); mask (nullable, 2D-CTC): strides (mN, mH, mW).  out int32 [N, W]. */
int mr_ctc_greedy_decode(const float *prob, const float *mask, int N, int C, int H, int W, int64_t sN, int64_t sC,
                         int64_t sH, int64_t sW, int64_t mN, int64_t mH, int64_t mW, int blank, int unknown, int *out,
                         void *stream) {
    if (N < 0 || C <= 0 || H <= 0 || W <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!prob || !out) return MR_ERR_NULL_POINTER;
    if ((size_t)W * sizeof(int) > 48 * 1024) return MR_ERR_UNSUPPORTED;
    const int threads = W < 32 ? 32 : (W > 256 ? 256 : (int)round_up(W, 32));
    ctc_greedy_decode_kernel<<<N, threads, (size_t)W * sizeof(int), (cudaStream_t)stream>>>(prob, mask, C, H, W, sN, sC, sH, sW,
                                                                                        mN, mH, mW, blank, unknown, out);
    return check_launch("ctc_greedy_decode_kernel");
}

int mr_blank_after_first_blank(int *pred, int N, int W, int blank, void *stream) {
    if (N < 0 || W <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!pred) return MR_ERR_NULL_POINTER;
    blank_after_first_blank_kernel<<<(int)ceil_div(N, 128), 128, 0, (cudaStream_t)stream>>>(pred, N, W, blank);
    return check_launch("blank_after_first_blank_kernel");
}

/* Conv weight [Cout,Cin,kh,kw] fp32 -> GEMM operand in `dtype` (0 fp32, 1 bf16): mode 0 forward matrix [Cout, Kp]
 * (column (i*kw+j)*Cp + c, zero padded), mode 1 input-gradient matrix [Cin, kh*kw*Cout] (taps flipped, transposed). */
int mr_conv_weight_pack(const float *w, int Cout, int Cin, int kh, int kw, int Cp, int Kp, int mode, int dtype, void *out,
                        void *stream) {
    if (Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0 || Cp < Cin || Kp < kh * kw * Cp || (mode != 0 && mode != 1)) return MR_ERR_BAD_SHAPE;
    if (!w || !out) return MR_ERR_NULL_POINTER;
    const int64_t total = mode == 0 ? (int64_t)Cout * Kp : (int64_t)Cin * kh * kw * Cout;
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH(dtype, (conv_weight_pack_kernel<T><<<grid1d(total, 256, 8), 256, 0, st>>>(w, Cout, Cin, kh, kw, Cp, Kp, mode, (T *)out)));
    return check_launch("conv_weight_pack_kernel");
}

/* LSTM gate rows: out[r,:] = a[src(r),:] (+ b[src(r),:]) for a [4H, cols] fp32; inverse = 0 gate-major -> unit-major
 * (row 4j+g <- row gH+j), inverse = 1 the way back; out in `dtype`. */
int mr_gate_rows_permute(const float *a, const float *b, int H, int cols, int inverse, int dtype, void *out, void *stream) {
    if (H <= 0 || cols <= 0) return MR_ERR_BAD_SHAPE;
    if (!a || !out) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH(dtype, (gate_rows_permute_kernel<T><<<grid1d((int64_t)4 * H * cols, 256, 8), 256, 0, st>>>(a, b, H, cols, inverse, (T *)out)));
    return check_launch("gate_rows_permute_kernel");
}

}  // extern "C"
