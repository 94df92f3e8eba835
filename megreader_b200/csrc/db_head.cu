// DB (Differentiable Binarization) text-detector tail: decoders/seg_detector.py:146-147 and 189-191, and the whole
// L1BalanceCELoss criterion (decoders/seg_detector_loss.py:162-185 with dice_loss.py:38-40, l1_loss.py:10,
// balance_cross_entropy_loss.py:40-52) as a fixed sequence of launches with no host synchronisation.
//
// Step function:   binary = sigmoid(zb), thresh = sigmoid(zt), thresh_binary = 1 / (1 + exp(-k (binary - thresh)))
//
// Loss.  Maps binary / thresh / thresh_binary / gt are [N,1,H,W], mask / thresh_map / thresh_mask are [N,H,W].  As in the
// reference, the balanced cross entropy multiplies the [N,1,H,W] gt with the [N,H,W] mask, which broadcasts to [N,N,H,W]:
//     pos[i,j,p] = trunc(gt[i,p] * mask[j,p]),  neg[i,j,p] = trunc((1 - gt[i,p]) * mask[j,p]),  bce[j,p] = BCE(binary[j,p], gt[j,p])
//     positive_loss = sum bce[j,p] * pos[i,j,p]
//     k             = min(sum neg, int(sum pos * negative_ratio))
//     topk_sum      = sum of the k largest of v[i,j,p] = bce[j,p] * neg[i,j,p]            (N*N*H*W values, zeros included)
//     bce_loss      = (positive_loss + topk_sum) / (sum pos + k + bce_eps)
// For N = 1 this is the per-pixel formula.  No value array is stored: every pass recomputes v from (binary, gt, mask) with the
// same rounded operations, one thread per pixel position p holding the N gt values of its column in shared memory.
//
// Top-k sum without the host: a radix select over the order-preserving 32-bit keys of v (8-bit digits, most significant first).
// Each digit is one histogram pass (block histograms in shared memory, integer atomics into global) followed by a one-CTA scan that
// picks the digit bin holding the k-th largest value and updates (prefix, k remaining, count above) in device memory.  After four
// digits the prefix is the key of tau, the k-th largest value, and cnt_gt the number of values above it; then
//     topk_sum = sum(v > tau) + (k - cnt_gt) * tau,
// which is the value torch.topk(...).sum() returns, ties included.  Floating-point sums use a grid fixed by H*W and a fixed-order
// final reduction (double accumulators), so results are bit-identical run to run and independent of the device's SM count.
// Backward gives negatives tied at tau the weight (k - cnt_gt) / cnt_eq each (DESIGN.md section 7).
#include "common.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

namespace {
using namespace mr;

constexpr int kThreads = 128;          // pixel positions per block in the loss kernels
constexpr int kMaxGrid = 2048;         // loss-kernel grid = min(ceil(HW / kThreads), kMaxGrid): depends on H*W only
constexpr int kMaxN = 192;             // the gt column of a block lives in shared memory: N * kThreads floats
constexpr int kScanThreads = 256;

struct DbState {
    double pos_loss, l1_num, l1_den, inter, uni, sum_gt;
    unsigned long long pos_cnt, neg_cnt, k, k_rem, cnt_gt, cnt_eq;
    unsigned prefix, pmask;
    // saved for the backward pass
    double bce_denom;
    float tau, w_tie;
    unsigned tau_key, pad;
};
struct DbPartial {
    double pos_loss, l1_num, l1_den, inter, uni;
    unsigned long long pos_cnt, neg_cnt, pad;
};

inline int64_t loss_grid(int64_t HW) { return std::min<int64_t>(ceil_div(HW, kThreads), kMaxGrid); }
inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
inline size_t off_hist() { return align256(sizeof(DbState)); }
inline size_t off_part() { return off_hist() + align256(4 * 256 * sizeof(unsigned long long)); }
inline size_t off_sum(int64_t G) { return off_part() + align256(G * sizeof(DbPartial)); }
inline size_t ws_bytes(int64_t G) { return off_sum(G) + align256(G * sizeof(double)); }

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16(v); }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half(v); }

// torch.sigmoid and the reference's step function, operation by operation
__device__ __forceinline__ float sigmoid_f(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }
__device__ __forceinline__ float step_exp(float b, float t, float k) { return expf(__fmul_rn(-k, __fsub_rn(b, t))); }

// torch's binary_cross_entropy (reduction='none'): the log terms are clamped at -100.  Explicitly rounded operations, so the
// histogram, sum and backward passes recompute exactly the value of the first pass.
__device__ __forceinline__ float bce_f(float p, float y) {
    const float lp = fmaxf(logf(p), -100.f), l1p = fmaxf(log1pf(-p), -100.f);
    return __fsub_rn(__fmul_rn(__fsub_rn(y, 1.f), l1p), __fmul_rn(y, lp));
}
// order-preserving key of a float (-0 and +0 share the key of +0)
__device__ __forceinline__ unsigned fkey(float v) {
    unsigned u = __float_as_uint(v == 0.f ? 0.f : v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_f(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ float trunc_w(float a) { return truncf(a); }

// ---------------------------------------------------------------------------------------------------------------- step
template <typename T>
__global__ void db_step_fwd_kernel(const T *__restrict__ zb, const T *__restrict__ zt, int64_t n, float k,
                                   float *__restrict__ binary, float *__restrict__ thresh, float *__restrict__ thresh_binary) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float b = sigmoid_f(to_f(zb[i]));
        binary[i] = b;
        if (zt) {
            const float t = sigmoid_f(to_f(zt[i]));
            thresh[i] = t;
            thresh_binary[i] = __fdiv_rn(1.f, __fadd_rn(1.f, step_exp(b, t, k)));
        }
    }
}

// reference autograd chain: sigmoid backward g*y*(1-y); d s / d b = k * r^2 * e with r = 1/(1+e), e = exp(-k (b - t))
template <typename T>
__global__ void db_step_bwd_kernel(const float *__restrict__ binary, const float *__restrict__ thresh,
                                   const float *__restrict__ thresh_binary, const float *__restrict__ gb,
                                   const float *__restrict__ gt_, const float *__restrict__ gs, int64_t n, float k,
                                   T *__restrict__ dzb, T *__restrict__ dzt) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float b = binary[i];
        float db = gb ? gb[i] : 0.f;
        if (dzt) {
            const float t = thresh[i];
            float dt = gt_ ? gt_[i] : 0.f;
            if (gs) {
                const float r = thresh_binary[i], e = step_exp(b, t, k);
                const float d = gs[i] * r * r * e * k;
                db += d;
                dt -= d;
            }
            dzt[i] = from_f<T>(dt * t * (1.f - t));
        }
        dzb[i] = from_f<T>(db * b * (1.f - b));
    }
}

// ---------------------------------------------------------------------------------------------------------------- loss
struct LossArgs {
    const float *binary, *thresh, *thresh_binary, *gt, *mask, *thresh_map, *thresh_mask;
    int N;
    int64_t HW;
};

__device__ __forceinline__ void load_gt_column(const LossArgs &a, int64_t p, float *sg) {
    for (int i = 0; i < a.N; ++i) sg[i * kThreads + threadIdx.x] = p < a.HW ? a.gt[i * a.HW + p] : 0.f;
}

// Visit the N values v[i,j,p] of (j, p) as runs of equal keys: f(key, count).  The common case (hard gt, mask in {0,1})
// is two runs at most, which keeps the shared-memory atomics per pixel close to one.
template <typename F>
__device__ __forceinline__ void for_value_runs(int N, const float *sg, float loss_j, float m_j, F &&f) {
    unsigned cur = 0;
    unsigned run = 0;
    for (int i = 0; i < N; ++i) {
        const float w = trunc_w(__fmul_rn(__fsub_rn(1.f, sg[i * kThreads + threadIdx.x]), m_j));
        const unsigned key = fkey(__fmul_rn(loss_j, w));
        if (run && key == cur) { ++run; continue; }
        if (run) f(cur, run);
        cur = key;
        run = 1;
    }
    if (run) f(cur, run);
}

__device__ __forceinline__ double block_sum_d(double v, double *red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[w] = v;
    __syncthreads();
    double s = 0.0;
    for (int i = 0; i < nw; ++i) s += red[i];
    return s;
}
__device__ __forceinline__ unsigned long long block_sum_u(unsigned long long v, unsigned long long *red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[w] = v;
    __syncthreads();
    unsigned long long s = 0;
    for (int i = 0; i < nw; ++i) s += red[i];
    return s;
}

// Pass 1: per-block partial sums of every reduction of the loss, and the histogram of the top key digit of all N*N*H*W values.
__global__ void __launch_bounds__(kThreads) db_loss_pass1_kernel(LossArgs a, DbPartial *__restrict__ part,
                                                                 unsigned long long *__restrict__ hist) {
    extern __shared__ float sg[];
    __shared__ unsigned sh[256];
    __shared__ double redd[kThreads / 32];
    __shared__ unsigned long long redu[kThreads / 32];
    for (int b = threadIdx.x; b < 256; b += kThreads) sh[b] = 0;
    double pos_loss = 0, l1n = 0, l1d = 0, inter = 0, uni = 0;
    unsigned long long pc = 0, nc = 0;
    __syncthreads();
    for (int64_t base = (int64_t)blockIdx.x * kThreads; base < a.HW; base += (int64_t)gridDim.x * kThreads) {
        const int64_t p = base + threadIdx.x;
        __syncthreads();
        load_gt_column(a, p, sg);
        __syncthreads();
        if (p >= a.HW) continue;
        for (int j = 0; j < a.N; ++j) {
            const int64_t q = j * a.HW + p;
            const float y = sg[j * kThreads + threadIdx.x], m = a.mask[q];
            const float l = bce_f(a.binary[q], y);
            // dice on thresh_binary, L1 on thresh (per pixel, no broadcast)
            const float tb = a.thresh_binary[q], tm = a.thresh_mask[q];
            inter += (double)__fmul_rn(__fmul_rn(tb, y), m);
            uni += (double)__fmul_rn(tb, m) + (double)__fmul_rn(y, m);
            l1n += (double)__fmul_rn(fabsf(__fsub_rn(a.thresh[q], a.thresh_map[q])), tm);
            l1d += (double)tm;
            for (int i = 0; i < a.N; ++i) {
                const float wp = trunc_w(__fmul_rn(sg[i * kThreads + threadIdx.x], m));
                const float wn = trunc_w(__fmul_rn(__fsub_rn(1.f, sg[i * kThreads + threadIdx.x]), m));
                pos_loss += (double)__fmul_rn(l, wp);
                pc += (unsigned long long)wp;
                nc += (unsigned long long)wn;
            }
            for_value_runs(a.N, sg, l, m, [&](unsigned key, unsigned cnt) { atomicAdd(&sh[key >> 24], cnt); });
        }
    }
    DbPartial r;
    r.pos_loss = block_sum_d(pos_loss, redd);
    r.l1_num = block_sum_d(l1n, redd);
    r.l1_den = block_sum_d(l1d, redd);
    r.inter = block_sum_d(inter, redd);
    r.uni = block_sum_d(uni, redd);
    r.pos_cnt = block_sum_u(pc, redu);
    r.neg_cnt = block_sum_u(nc, redu);
    r.pad = 0;
    if (threadIdx.x == 0) part[blockIdx.x] = r;
    __syncthreads();
    for (int b = threadIdx.x; b < 256; b += kThreads)
        if (sh[b]) atomicAdd(&hist[b], (unsigned long long)sh[b]);
}

// Histogram of key digit `d` (bits 8d .. 8d+7) over the values whose higher digits equal the selected prefix.
__global__ void __launch_bounds__(kThreads) db_loss_hist_kernel(LossArgs a, int d, const DbState *__restrict__ st,
                                                                unsigned long long *__restrict__ hist) {
    extern __shared__ float sg[];
    __shared__ unsigned sh[256];
    for (int b = threadIdx.x; b < 256; b += kThreads) sh[b] = 0;
    const unsigned prefix = st->prefix, pmask = st->pmask;
    const int shift = 8 * d;
    __syncthreads();
    for (int64_t base = (int64_t)blockIdx.x * kThreads; base < a.HW; base += (int64_t)gridDim.x * kThreads) {
        const int64_t p = base + threadIdx.x;
        __syncthreads();
        load_gt_column(a, p, sg);
        __syncthreads();
        if (p >= a.HW) continue;
        for (int j = 0; j < a.N; ++j) {
            const int64_t q = j * a.HW + p;
            const float l = bce_f(a.binary[q], sg[j * kThreads + threadIdx.x]);
            for_value_runs(a.N, sg, l, a.mask[q], [&](unsigned key, unsigned cnt) {
                if ((key & pmask) == prefix) atomicAdd(&sh[(key >> shift) & 255u], cnt);
            });
        }
    }
    __syncthreads();
    for (int b = threadIdx.x; b < 256; b += kThreads)
        if (sh[b]) atomicAdd(&hist[b], (unsigned long long)sh[b]);
}

// One CTA.  d == 3: first reduce the pass-1 partials in a fixed order and compute k.  Then pick the bin of digit d that holds
// the k_rem-th largest of the remaining values.
__global__ void __launch_bounds__(kScanThreads) db_loss_scan_kernel(int d, int G, float negative_ratio,
                                                                    const DbPartial *__restrict__ part,
                                                                    const unsigned long long *__restrict__ hist,
                                                                    DbState *__restrict__ st) {
    __shared__ unsigned long long sh[256];
    __shared__ double red[kScanThreads / 32];
    __shared__ unsigned long long redu[kScanThreads / 32];
    if (d == 3) {
        double v[5] = {0, 0, 0, 0, 0};
        unsigned long long c[2] = {0, 0};
        for (int b = threadIdx.x; b < G; b += kScanThreads) {
            const DbPartial &r = part[b];
            v[0] += r.pos_loss; v[1] += r.l1_num; v[2] += r.l1_den; v[3] += r.inter; v[4] += r.uni;
            c[0] += r.pos_cnt; c[1] += r.neg_cnt;
        }
        for (int t = 0; t < 5; ++t) v[t] = block_sum_d(v[t], red);
        for (int t = 0; t < 2; ++t) c[t] = block_sum_u(c[t], redu);
        if (threadIdx.x == 0) {
            st->pos_loss = v[0]; st->l1_num = v[1]; st->l1_den = v[2]; st->inter = v[3]; st->uni = v[4];
            st->pos_cnt = c[0]; st->neg_cnt = c[1];
            // int(positive_count * negative_ratio): a double product truncated toward zero, as Python does
            const double lim = (double)c[0] * (double)negative_ratio;
            const unsigned long long kk = lim <= 0.0 ? 0ull : (unsigned long long)lim;
            st->k = kk < c[1] ? kk : c[1];
            st->k_rem = st->k;
            st->cnt_gt = 0;
            st->prefix = 0;
            st->pmask = 0;
        }
    }
    sh[threadIdx.x] = hist[threadIdx.x];
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned long long k_rem = st->k_rem;
        if (k_rem == 0) {                    // k = 0: nothing is selected; tau sits above every key
            st->prefix = 0xffffffffu;
            st->pmask = 0xffffffffu;
            st->cnt_eq = 1;
        } else {
            unsigned long long cum = 0;
            int b = 255;
            for (; b > 0; --b) {
                if (cum + sh[b] >= k_rem) break;
                cum += sh[b];
            }
            st->cnt_gt += cum;
            st->k_rem = k_rem - cum;
            st->prefix |= (unsigned)b << (8 * d);
            st->pmask |= 255u << (8 * d);
            st->cnt_eq = sh[b];
        }
    }
}

// sum of the values strictly above tau: per-block partials in double, reduced in fixed order by db_loss_final_kernel
__global__ void __launch_bounds__(kThreads) db_loss_sum_kernel(LossArgs a, const DbState *__restrict__ st, double *__restrict__ part) {
    extern __shared__ float sg[];
    __shared__ double red[kThreads / 32];
    const unsigned tau_key = st->prefix;
    const bool none = st->k == 0;
    double s = 0.0;
    for (int64_t base = (int64_t)blockIdx.x * kThreads; base < a.HW && !none; base += (int64_t)gridDim.x * kThreads) {
        const int64_t p = base + threadIdx.x;
        __syncthreads();
        load_gt_column(a, p, sg);
        __syncthreads();
        if (p >= a.HW) continue;
        for (int j = 0; j < a.N; ++j) {
            const int64_t q = j * a.HW + p;
            const float l = bce_f(a.binary[q], sg[j * kThreads + threadIdx.x]);
            for_value_runs(a.N, sg, l, a.mask[q], [&](unsigned key, unsigned cnt) {
                if (key > tau_key) s += (double)cnt * (double)key_f(key);
            });
        }
    }
    s = block_sum_d(s, red);
    if (threadIdx.x == 0) part[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kScanThreads) db_loss_final_kernel(int G, float eps_dice, float bce_eps, float l1_scale,
                                                                     float bce_scale, const double *__restrict__ part,
                                                                     DbState *__restrict__ st, float *__restrict__ out) {
    __shared__ double red[kScanThreads / 32];
    double s = 0.0;
    for (int b = threadIdx.x; b < G; b += kScanThreads) s += part[b];
    s = block_sum_d(s, red);
    if (threadIdx.x == 0) {
        const unsigned long long k = st->k;
        double topk = 0.0;
        float tau = 0.f, w_tie = 0.f;
        if (k) {
            tau = key_f(st->prefix);
            topk = s + (double)(k - st->cnt_gt) * (double)tau;
            w_tie = (float)((double)(k - st->cnt_gt) / (double)st->cnt_eq);
        }
        const double denom = (double)st->pos_cnt + (double)k + (double)bce_eps;
        const double bce = (st->pos_loss + topk) / denom;
        const double uni = st->uni + (double)eps_dice;
        const double dice = 1.0 - 2.0 * st->inter / uni;
        const double l1 = st->l1_num / st->l1_den;
        st->sum_gt = s;
        st->bce_denom = denom;
        st->tau = tau;
        st->w_tie = w_tie;
        st->tau_key = st->prefix;
        st->uni = uni;
        out[0] = (float)(dice + (double)l1_scale * l1 + (double)bce_scale * bce);
        out[1] = (float)bce;
        out[2] = (float)dice;
        out[3] = (float)l1;
    }
}

// grad_out = d(loss, bce_loss, dice_loss, l1_loss)
__global__ void __launch_bounds__(kThreads) db_loss_bwd_kernel(LossArgs a, float l1_scale, float bce_scale,
                                                               const DbState *__restrict__ st, const float *__restrict__ grad_out,
                                                               float *__restrict__ d_binary, float *__restrict__ d_thresh,
                                                               float *__restrict__ d_thresh_binary) {
    extern __shared__ float sg[];
    const float g0 = grad_out[0];
    const double g_bce = (double)g0 * bce_scale + grad_out[1], g_dice = (double)g0 + grad_out[2],
                 g_l1 = (double)g0 * l1_scale + grad_out[3];
    const float c_bce = (float)(g_bce / st->bce_denom);
    const float c_l1 = (float)(g_l1 / st->l1_den);
    const double U = st->uni;
    const float c_dice_g = (float)(-2.0 * g_dice / U), c_dice_i = (float)(2.0 * g_dice * st->inter / (U * U));
    const bool none = st->k == 0;
    const unsigned tau_key = st->tau_key;
    const float w_tie = st->w_tie;
    for (int64_t base = (int64_t)blockIdx.x * kThreads; base < a.HW; base += (int64_t)gridDim.x * kThreads) {
        const int64_t p = base + threadIdx.x;
        __syncthreads();
        load_gt_column(a, p, sg);
        __syncthreads();
        if (p >= a.HW) continue;
        for (int j = 0; j < a.N; ++j) {
            const int64_t q = j * a.HW + p;
            const float y = sg[j * kThreads + threadIdx.x], m = a.mask[q], pr = a.binary[q];
            const float l = bce_f(pr, y);
            float w = 0.f;
            for (int i = 0; i < a.N; ++i) {
                const float gi = sg[i * kThreads + threadIdx.x];
                w += trunc_w(__fmul_rn(gi, m));
                const float wn = trunc_w(__fmul_rn(__fsub_rn(1.f, gi), m));
                if (!none && wn != 0.f) {
                    const unsigned key = fkey(__fmul_rn(l, wn));
                    w += key > tau_key ? wn : (key == tau_key ? wn * w_tie : 0.f);
                }
            }
            // torch's binary_cross_entropy backward: (p - y) / max((1 - p) p, 1e-12)
            d_binary[q] = w == 0.f ? 0.f : c_bce * w * (pr - y) / fmaxf((1.f - pr) * pr, 1e-12f);
            const float diff = a.thresh[q] - a.thresh_map[q];
            const float sgn = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
            d_thresh[q] = c_l1 * sgn * a.thresh_mask[q];
            d_thresh_binary[q] = c_dice_g * y * m + c_dice_i * m;
        }
    }
}

int elem_grid(int64_t n) { return (int)std::min<int64_t>(ceil_div(n, 256), (int64_t)sm_count() * 16); }

bool loss_args_ok(const LossArgs &a) {
    return a.binary && a.thresh && a.thresh_binary && a.gt && a.mask && a.thresh_map && a.thresh_mask;
}

}  // namespace

extern "C" {

int mr_db_step_fwd(const void *zb, const void *zt, int dtype, int64_t n, float k, float *binary, float *thresh,
                   float *thresh_binary, void *stream) {
    if (n < 0 || dtype < 0 || dtype > 2) return MR_ERR_BAD_SHAPE;
    if (n == 0) return MR_OK;
    if (!zb || !binary || (zt && (!thresh || !thresh_binary))) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    const int g = elem_grid(n);
    if (dtype == 0)
        db_step_fwd_kernel<float><<<g, 256, 0, st>>>((const float *)zb, (const float *)zt, n, k, binary, thresh, thresh_binary);
    else if (dtype == 1)
        db_step_fwd_kernel<__nv_bfloat16><<<g, 256, 0, st>>>((const __nv_bfloat16 *)zb, (const __nv_bfloat16 *)zt, n, k, binary,
                                                             thresh, thresh_binary);
    else
        db_step_fwd_kernel<__half><<<g, 256, 0, st>>>((const __half *)zb, (const __half *)zt, n, k, binary, thresh, thresh_binary);
    return check_launch("db_step_fwd");
}

int mr_db_step_bwd(const float *binary, const float *thresh, const float *thresh_binary, const float *g_binary,
                   const float *g_thresh, const float *g_thresh_binary, int dtype, int64_t n, float k, void *d_zb, void *d_zt,
                   void *stream) {
    if (n < 0 || dtype < 0 || dtype > 2) return MR_ERR_BAD_SHAPE;
    if (n == 0) return MR_OK;
    if (!binary || !d_zb || (d_zt && !thresh) || (d_zt && g_thresh_binary && !thresh_binary)) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    const int g = elem_grid(n);
    if (dtype == 0)
        db_step_bwd_kernel<float><<<g, 256, 0, st>>>(binary, thresh, thresh_binary, g_binary, g_thresh, g_thresh_binary, n, k,
                                                     (float *)d_zb, (float *)d_zt);
    else if (dtype == 1)
        db_step_bwd_kernel<__nv_bfloat16><<<g, 256, 0, st>>>(binary, thresh, thresh_binary, g_binary, g_thresh, g_thresh_binary, n,
                                                             k, (__nv_bfloat16 *)d_zb, (__nv_bfloat16 *)d_zt);
    else
        db_step_bwd_kernel<__half><<<g, 256, 0, st>>>(binary, thresh, thresh_binary, g_binary, g_thresh, g_thresh_binary, n, k,
                                                      (__half *)d_zb, (__half *)d_zt);
    return check_launch("db_step_bwd");
}

int64_t mr_db_loss_workspace_bytes(int64_t N, int64_t H, int64_t W) {
    if (N <= 0 || H <= 0 || W <= 0) return 0;
    return (int64_t)ws_bytes(loss_grid(H * W));
}

int mr_db_loss_fwd_f32(const float *binary, const float *thresh, const float *thresh_binary, const float *gt, const float *mask,
                       const float *thresh_map, const float *thresh_mask, int N, int H, int W, float eps, float bce_eps,
                       float l1_scale, float bce_scale, float negative_ratio, void *workspace, float *out_scalars, void *stream) {
    if (N <= 0 || H <= 0 || W <= 0) return MR_ERR_BAD_SHAPE;
    if (N > kMaxN) return MR_ERR_UNSUPPORTED;
    LossArgs a{binary, thresh, thresh_binary, gt, mask, thresh_map, thresh_mask, N, (int64_t)H * W};
    if (!loss_args_ok(a) || !workspace || !out_scalars) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    const int G = (int)loss_grid(a.HW);
    char *ws = (char *)workspace;
    DbState *state = (DbState *)ws;
    unsigned long long *hist = (unsigned long long *)(ws + off_hist());
    DbPartial *part = (DbPartial *)(ws + off_part());
    double *sums = (double *)(ws + off_sum(G));
    const size_t smem = (size_t)N * kThreads * sizeof(float);
    int rc;
    if ((rc = ensure_dyn_smem((const void *)db_loss_pass1_kernel, smem, "db_loss smem"))) return rc;
    if ((rc = ensure_dyn_smem((const void *)db_loss_hist_kernel, smem, "db_loss smem"))) return rc;
    if ((rc = ensure_dyn_smem((const void *)db_loss_sum_kernel, smem, "db_loss smem"))) return rc;
    MR_CUDA_TRY(cudaMemsetAsync(hist, 0, 4 * 256 * sizeof(unsigned long long), st), "db_loss memset");
    db_loss_pass1_kernel<<<G, kThreads, smem, st>>>(a, part, hist + 3 * 256);
    if ((rc = check_launch("db_loss_pass1"))) return rc;
    db_loss_scan_kernel<<<1, kScanThreads, 0, st>>>(3, G, negative_ratio, part, hist + 3 * 256, state);
    if ((rc = check_launch("db_loss_scan"))) return rc;
    for (int d = 2; d >= 0; --d) {
        db_loss_hist_kernel<<<G, kThreads, smem, st>>>(a, d, state, hist + d * 256);
        if ((rc = check_launch("db_loss_hist"))) return rc;
        db_loss_scan_kernel<<<1, kScanThreads, 0, st>>>(d, G, negative_ratio, part, hist + d * 256, state);
        if ((rc = check_launch("db_loss_scan"))) return rc;
    }
    db_loss_sum_kernel<<<G, kThreads, smem, st>>>(a, state, sums);
    if ((rc = check_launch("db_loss_sum"))) return rc;
    db_loss_final_kernel<<<1, kScanThreads, 0, st>>>(G, eps, bce_eps, l1_scale, bce_scale, sums, state, out_scalars);
    return check_launch("db_loss_final");
}

int mr_db_loss_bwd_f32(const float *binary, const float *thresh, const float *thresh_binary, const float *gt, const float *mask,
                       const float *thresh_map, const float *thresh_mask, int N, int H, int W, float l1_scale, float bce_scale,
                       const void *workspace, const float *grad_out, float *d_binary, float *d_thresh, float *d_thresh_binary,
                       void *stream) {
    if (N <= 0 || H <= 0 || W <= 0) return MR_ERR_BAD_SHAPE;
    if (N > kMaxN) return MR_ERR_UNSUPPORTED;
    LossArgs a{binary, thresh, thresh_binary, gt, mask, thresh_map, thresh_mask, N, (int64_t)H * W};
    if (!loss_args_ok(a) || !workspace || !grad_out || !d_binary || !d_thresh || !d_thresh_binary) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = (size_t)N * kThreads * sizeof(float);
    int rc;
    if ((rc = ensure_dyn_smem((const void *)db_loss_bwd_kernel, smem, "db_loss smem"))) return rc;
    const int G = (int)std::min<int64_t>(ceil_div(a.HW, kThreads), (int64_t)sm_count() * 16);
    db_loss_bwd_kernel<<<G, kThreads, smem, st>>>(a, l1_scale, bce_scale, (const DbState *)workspace, grad_out, d_binary,
                                                   d_thresh, d_thresh_binary);
    return check_launch("db_loss_bwd");
}

}  // extern "C"
