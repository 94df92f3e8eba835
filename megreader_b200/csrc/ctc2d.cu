// 2D-CTC loss for sm_90a — forward (log_alpha + nll), backward (gradient), and the training pair
// (forward_train + backward_apply).  Replaces the reference's four SIMT kernels
// (ops/ctc_2d/csrc/cuda/ctc2d_cuda_kernel.cu:54-211 K1, :254-368 K2, :427-517 K3) — not a port:
//
// Observation that shapes the design.  In the reference recurrence every height shares one
// transition term:  alpha[t,h,s] = lp[t,h,l'_s] + R[t,s]  with
//     R[t,s]   = LSE( A[t-1,s], A[t-1,s-1], [l'_s != l'_{s-2}] A[t-1,s-2] )
//     A[t,s]   = LSE_h alpha[t,h,s] = R[t,s] + Q[t,l'_s],      Q[t,c] = LSE_h lp[t,h,c]
// so the dynamic programme is a 1D CTC over the height-marginal Q (tiny, on chip), and log_alpha is a
// pure streaming expansion of lp.  Likewise beta[t,h,s] = lp[t,h,l'_s] + Rb[t,s], and K3's gradient
//     grad[t,h,c] = (exp(lp) - exp(LSE_{s:l'_s=c}(alpha+beta) + nll - lp)) * go
//                 = exp(lp[t,h,c]) * (1 - sum_{s:l'_s=c} exp(R[t,s] + Rb[t,s] + nll)) * go      (class present)
// needs only a per-(t,c) factor.  Hence: log_probs is read ONCE per kernel, log_beta never exists in
// HBM, and the backward never reads log_alpha.
//
// Kernels (all HBM-bound; algorithmic bytes per sample, fp32, cfg-3 shape T32 H8 C38 S32):
//   ctc2d_alpha_kernel   : read |lp| 38,912 + write |alpha| 66,560            (contract forward)
//   ctc2d_dp_kernel<GRAD>: read |lp| (+ L2 re-read) + write |grad| 38,912      (contract backward)
//   ctc2d_dp_kernel<FAC> : read |lp| + write gfac T*C*4 = 4,864                (training forward)
//   ctc2d_apply_kernel   : read |lp| + gfac, write |grad|                      (training backward)
#include "common.cuh"
#include <math.h>
#include <string.h>
#include <stdlib.h>

namespace {

using namespace mr;

constexpr int kStages = 4;  // cp.async ring depth of the alpha kernel

template <typename real> struct Lim;
template <> struct Lim<float> { static __device__ __forceinline__ float ninf() { return -INFINITY; } };
template <> struct Lim<double> { static __device__ __forceinline__ double ninf() { return -(double)INFINITY; } };

// fast path: one FMUL + one MUFU each (ex2/lg2.approx.ftz).  __expf/__logf without -use_fast_math expand to
// denormal-safe sequences (FSETP + 2 extra FMUL), a large share of the DP kernel's instructions; flushing results below 1.2e-38 to zero is harmless in a log-sum-exp.
__device__ __forceinline__ float ex2_ftz(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_ftz(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
template <bool FAST> __device__ __forceinline__ float ex(float x) { return FAST ? ex2_ftz(x * 1.4426950408889634f) : expf(x); }
template <bool FAST> __device__ __forceinline__ float lg(float x) { return FAST ? lg2_ftz(x) * 0.6931471805599453f : logf(x); }
template <bool FAST> __device__ __forceinline__ double ex(double x) { return exp(x); }
template <bool FAST> __device__ __forceinline__ double lg(double x) { return log(x); }

// LSE with the all -inf case returning -inf (safe_log_add, ctc2d_cuda_kernel.cu:44-51 / :166-167)
template <bool FAST, typename real>
__device__ __forceinline__ real lse2(real a, real b) {
    real m = fmax(a, b);
    if (m == Lim<real>::ninf()) return m;
    return m + lg<FAST>(ex<FAST>(a - m) + ex<FAST>(b - m));
}
template <bool FAST, typename real>
__device__ __forceinline__ real lse3(real a, real b, real c) {
    real m = fmax(a, fmax(b, c));
    if (m == Lim<real>::ninf()) return m;
    return m + lg<FAST>(ex<FAST>(a - m) + ex<FAST>(b - m) + ex<FAST>(c - m));
}

struct Geo {
    int T, H, N, C, S, SS;  // SS = 2S+1
    int G;                  // samples per CTA
    int vec;                // elements per 16-byte vector usable on log_probs rows (1 = scalar path)
    int blank;
    int zero_inf;           // MODE_FAC_STD: zero the factor of samples whose nll is +inf (zero_infinity=True)
    int64_t tg_sn, tg_ss;
};

__device__ __forceinline__ int clampi(int64_t v, int hi) { return v < 0 ? 0 : (v >= hi ? hi - 1 : (int)v); }

// Per-thread view of one (sample, state): lengths, l'_s and the skip flags (K1 :113-123, K2 :304-314).
struct StateCtx {
    bool active;
    int g, s, b, cur;
    int64_t Tb, L;
    bool skip_fwd, skip_bwd, in_range;  // in_range: L > 0 && s <= 2L
};
__device__ __forceinline__ StateCtx make_ctx(const Geo &q, int b0, int Gv, const int64_t *tg, const int64_t *il,
                                             const int64_t *tl) {
    StateCtx c;
    const int tid = threadIdx.x;
    c.g = tid / q.SS;
    c.s = tid - c.g * q.SS;
    c.active = (tid < q.G * q.SS) && (c.g < Gv);
    c.b = b0 + c.g;
    c.cur = q.blank;
    c.Tb = 0; c.L = 0;
    c.skip_fwd = c.skip_bwd = c.in_range = false;
    if (c.active) {
        c.Tb = il[c.b];
        c.L = tl[c.b];
        if (c.s < 2 * c.L + 1) {
            c.in_range = c.L > 0;
            const int64_t *row = tg + (int64_t)c.b * q.tg_sn;
            if (c.s & 1) {
                const int64_t me = row[(int64_t)(c.s >> 1) * q.tg_ss];
                c.cur = clampi(me, q.C);
                if (c.s > 1) c.skip_fwd = row[(int64_t)((c.s - 2) >> 1) * q.tg_ss] != me;
                if (c.s < 2 * c.L - 1) c.skip_bwd = row[(int64_t)((c.s + 2) >> 1) * q.tg_ss] != me;
            }
        }
    }
    return c;
}

// ------------------------------------------------------------------------------------------------
// Contract forward: log_alpha + nll.  One CTA = G consecutive samples, thread = (sample, state).
// The [H, G*C] slab of log_probs for column t is prefetched kStages-1 columns ahead with cp.async;
// it feeds both Q[t] and the expansion, so HBM sees every byte of log_probs exactly once.
// All per-thread addressing (copy plan, output pointer, gather offset) is hoisted out of the column
// loop: index arithmetic otherwise takes most of the issue slots.
// ------------------------------------------------------------------------------------------------
constexpr int kPlan = 4;  // cp.async chunks per thread per column held in registers

template <typename real, bool FAST, bool STAGED, int HT>
__global__ void ctc2d_alpha_kernel(Geo q, const real *__restrict__ lp, const int64_t *__restrict__ tg,
                                   const int64_t *__restrict__ il, const int64_t *__restrict__ tl,
                                   real *__restrict__ nll, real *__restrict__ la) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const real NINF = Lim<real>::ninf();
    const int H = HT > 0 ? HT : q.H;
    const int tid = threadIdx.x, nth = blockDim.x;
    const int b0 = blockIdx.x * q.G;
    const int Gv = min(q.G, q.N - b0);
    const int rowElems = q.G * q.C;
    const int slabElems = H * rowElems;
    real *slab = reinterpret_cast<real *>(smem_raw);
    real *Qs = slab + (STAGED ? kStages * slabElems : 0);
    real *As = Qs + rowElems;
    real *fin = As + q.G * q.SS;
    const int64_t strideH = (int64_t)q.N * q.C;
    const int64_t strideT = strideH * H;
    const real *lp_cta = lp + (int64_t)b0 * q.C;

    const StateCtx c = make_ctx(q, b0, Gv, tg, il, tl);
    if (tid < 2 * q.G) fin[tid] = NINF;
    real R = NINF;

    // ---- copy plan: which chunks of a column slab this thread fetches (same for every column)
    int64_t pl_src[kPlan];
    int pl_dst[kPlan], pl_kind[kPlan];  // 0 none, 1 element, 2 16-byte vector
    bool plan_ok = false;
    const int n_el = Gv * q.C;
    const int nvec = n_el / q.vec, rem = n_el - nvec * q.vec, per_row = nvec + rem;
    if (STAGED) {
        plan_ok = H * per_row <= kPlan * nth;
#pragma unroll
        for (int m = 0; m < kPlan; ++m) {
            const int i = tid + m * nth;
            pl_kind[m] = 0; pl_src[m] = 0; pl_dst[m] = 0;
            if (i < H * per_row) {
                const int h = i / per_row, j = i - h * per_row;
                const int e = j < nvec ? j * q.vec : nvec * q.vec + (j - nvec);
                pl_kind[m] = (j < nvec && q.vec > 1) ? 2 : 1;
                pl_src[m] = h * strideH + e;
                pl_dst[m] = h * rowElems + e;
            }
        }
    }
    auto fetch = [&](int t, real *dst) {
        const real *base = lp_cta + t * strideT;
        if (plan_ok) {
#pragma unroll
            for (int m = 0; m < kPlan; ++m) {
                if (pl_kind[m] == 2) cp_async16(dst + pl_dst[m], base + pl_src[m]);
                else if (pl_kind[m] == 1) {
                    if (sizeof(real) == 8) cp_async8(dst + pl_dst[m], base + pl_src[m]);
                    else cp_async4(dst + pl_dst[m], base + pl_src[m]);
                }
            }
        } else {
            for (int i = tid; i < H * per_row; i += nth) {
                const int h = i / per_row, j = i - h * per_row;
                const int e = j < nvec ? j * q.vec : nvec * q.vec + (j - nvec);
                const real *src = base + h * strideH + e;
                real *d = dst + h * rowElems + e;
                if (j < nvec && q.vec > 1) cp_async16(d, src);
                else if (sizeof(real) == 8) cp_async8(d, src);
                else cp_async4(d, src);
            }
        }
    };

    if (STAGED) {
        for (int st = 0; st < kStages - 1; ++st) {
            if (st < q.T) fetch(st, slab + st * slabElems);
            cp_async_commit();
        }
    }
    const int gc = c.g * q.C + c.cur;                      // gather offset of l'_s inside a slab row
    real *out = la + ((int64_t)c.b * q.T * H) * q.SS + c.s;  // log_alpha[b, 0, 0, s]
    const int outT = H * q.SS;
    const real *arow = As + tid;                            // tid == g*SS + s for active threads

    for (int t = 0; t < q.T; ++t) {
        if (STAGED) cp_async_wait<kStages - 2>();
        __syncthreads();  // slab[t] landed; As/fin of column t-1 visible; slab[t-1] free for reuse
        if (STAGED) {
            const int tn = t + kStages - 1;
            if (tn < q.T) fetch(tn, slab + (tn % kStages) * slabElems);
            cp_async_commit();
        }
        if (c.active) {
            if (t == 0) {
                R = (c.s == 0 || (c.s == 1 && c.L > 0)) ? (real)0 : NINF;  // K1 :84-111
            } else if (t < c.Tb && c.in_range) {                           // K1 :128-173
                R = lse3<FAST>(arow[0], c.s > 0 ? arow[-1] : NINF, c.skip_fwd ? arow[-2] : NINF);
            } else {
                R = NINF;                                                  // K1 :174-182
            }
        }
        if (STAGED) {
            const real *sl = slab + (t % kStages) * slabElems;
            if (c.active) {
                const real *src = sl + gc;
#pragma unroll
                for (int h = 0; h < (HT > 0 ? HT : 1); ++h) {
                    if (HT > 0) __stcs(out + h * q.SS, src[h * rowElems] + R);
                }
                if (HT == 0)
                    for (int h = 0; h < H; ++h) __stcs(out + h * q.SS, src[h * rowElems] + R);
            }
            // Q[t][g][c] = LSE_h lp[t,h,b,c]
            for (int idx = tid; idx < n_el; idx += nth) {
                const real *p = sl + idx;
                real v;
                if (HT > 0) {
                    real x[HT > 0 ? HT : 1];
#pragma unroll
                    for (int h = 0; h < (HT > 0 ? HT : 1); ++h) x[h] = p[h * rowElems];
                    real m = x[0];
#pragma unroll
                    for (int h = 1; h < (HT > 0 ? HT : 1); ++h) m = fmax(m, x[h]);
                    v = m;
                    if (m != NINF) {
                        real sum = 0;
#pragma unroll
                        for (int h = 0; h < (HT > 0 ? HT : 1); ++h) sum += ex<FAST>(x[h] - m);
                        v = m + lg<FAST>(sum);
                    }
                } else {
                    real m = NINF;
                    for (int h = 0; h < H; ++h) m = fmax(m, p[h * rowElems]);
                    v = m;
                    if (m != NINF) {
                        real sum = 0;
                        for (int h = 0; h < H; ++h) sum += ex<FAST>(p[h * rowElems] - m);
                        v = m + lg<FAST>(sum);
                    }
                }
                Qs[idx] = v;
            }
        } else {
            const real *sl = lp_cta + t * strideT;
            if (c.active) {
                const real *src = sl + gc;
                for (int h = 0; h < H; ++h) __stcs(out + h * q.SS, src[h * strideH] + R);
            }
            for (int idx = tid; idx < n_el; idx += nth) {
                const real *p = sl + idx;
                real m = NINF;
                for (int h = 0; h < H; ++h) m = fmax(m, p[h * strideH]);
                real v = m;
                if (m != NINF) {
                    real sum = 0;
                    for (int h = 0; h < H; ++h) sum += ex<FAST>(p[h * strideH] - m);
                    v = m + lg<FAST>(sum);
                }
                Qs[idx] = v;
            }
        }
        out += outT;
        __syncthreads();
        if (c.active) {
            const real a = R + Qs[gc];
            As[tid] = a;
            if (t == c.Tb - 1) {  // K1 :189-209 reads LSE_h alpha[Tb-1, h, 2L] and [.., 2L-1]
                if (c.s == 2 * c.L) fin[2 * c.g] = a;
                else if (c.s == 2 * c.L - 1) fin[2 * c.g + 1] = a;
            }
        }
    }
    __syncthreads();
    if (c.active && c.s == 0) nll[c.b] = -lse2<FAST>(fin[2 * c.g], fin[2 * c.g + 1]);
}

// ------------------------------------------------------------------------------------------------
// DP kernel (contract backward / training forward).
//   P1  stream log_probs, Q[t][g][c] for all t into shared memory
//   P2  forward sweep R[t] (kept in smem), nll; backward sweep Rb[t] fused with the per-class
//       accumulation  acc[t][g][c] += exp(R + Rb + nll)   and the "class present" flag
//   P3  MODE_GRAD: re-stream log_probs (L2) and write grad = exp(lp) * fac * go
//       MODE_FAC : write fac [T,N,C] (+ nll)
// ------------------------------------------------------------------------------------------------
enum { MODE_GRAD = 0, MODE_FAC = 1, MODE_FAC_STD = 2 };  // FAC_STD: torch.nn.CTCLoss gradient convention (1D CTC)

template <typename real, int VE> struct alignas(sizeof(real) * VE) VecT { real v[VE]; };

// 4/8/16-byte vector loads/stores through the builtin types (so the cache-hint intrinsics apply)
template <int BYTES> struct Raw;
template <> struct Raw<16> { using type = float4; };
template <> struct Raw<8> { using type = float2; };
template <> struct Raw<4> { using type = float; };
template <typename real, int VE>
__device__ __forceinline__ VecT<real, VE> ld_nc(const real *p) {
    using R = typename Raw<sizeof(real) * VE>::type;
    const R t = __ldg(reinterpret_cast<const R *>(p));
    VecT<real, VE> r;
    memcpy(&r, &t, sizeof(R));
    return r;
}
template <typename real, int VE>
__device__ __forceinline__ VecT<real, VE> ld_cs(const real *p) {
    using R = typename Raw<sizeof(real) * VE>::type;
    const R t = __ldcs(reinterpret_cast<const R *>(p));
    VecT<real, VE> r;
    memcpy(&r, &t, sizeof(R));
    return r;
}
template <typename real, int VE>
__device__ __forceinline__ void st_cs(real *p, const VecT<real, VE> &v) {
    using R = typename Raw<sizeof(real) * VE>::type;
    R t;
    memcpy(&t, &v, sizeof(R));
    __stcs(reinterpret_cast<R *>(p), t);
}

// LSE over the H rows of one vector column, H processed in register chunks of 8.
template <typename real, bool FAST, int VE, int HT, bool LOG2OUT = false>
__device__ __forceinline__ void lse_rows(const real *base, int64_t hs, int H, real *dst) {
    const real NINF = Lim<real>::ninf();
    real m[VE], sum[VE];
#pragma unroll
    for (int k = 0; k < VE; ++k) { m[k] = NINF; sum[k] = 0; }
    for (int h0 = 0; h0 < H; h0 += 8) {
        VecT<real, VE> x[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            if ((HT > 0 && h0 + u < HT) || (HT == 0 && h0 + u < H)) x[u] = ld_nc<real, VE>(base + (h0 + u) * hs);
            else {
#pragma unroll
                for (int k = 0; k < VE; ++k) x[u].v[k] = NINF;
            }
        }
#pragma unroll
        for (int k = 0; k < VE; ++k) {
            real cm = x[0].v[k];
#pragma unroll
            for (int u = 1; u < 8; ++u) cm = fmax(cm, x[u].v[k]);
            const real nm = fmax(m[k], cm);
            if (nm != NINF) {
                real sacc = (m[k] == NINF) ? (real)0 : sum[k] * ex<FAST>(m[k] - nm);
#pragma unroll
                for (int u = 0; u < 8; ++u) sacc += ex<FAST>(x[u].v[k] - nm);
                sum[k] = sacc;
                m[k] = nm;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < VE; ++k) {
        if (LOG2OUT) dst[k] = (m[k] == NINF) ? NINF : (real)(m[k] * (real)1.4426950408889634 + (real)lg2_ftz((float)sum[k]));
        else dst[k] = (m[k] == NINF) ? NINF : m[k] + lg<FAST>(sum[k]);
    }
}

template <typename real, bool FAST, int VE, int HT, bool LOG2OUT = false>
__device__ __forceinline__ void phase_q(const Geo &q, const real *__restrict__ lp, real *Qall, int b0, int Gv, int pitch = 0) {
    const int H = HT > 0 ? HT : q.H;
    const int rowElems = pitch > 0 ? pitch : q.G * q.C;
    const int nvec = (Gv * q.C + VE - 1) / VE;  // VE > 1 only when Gv*C % VE == 0 for every CTA
    const int64_t hs = (int64_t)q.N * q.C;
    const int tid = threadIdx.x, nth = blockDim.x;
    const real *cta = lp + (int64_t)b0 * q.C;
    if (nvec <= nth) {  // thread-fixed vector column, stride over t: no per-item division
        const int tpr = nth / nvec;
        const int t0 = tid / nvec, j = tid - t0 * nvec;
        if (t0 < tpr) {
            int t = t0;
            for (; t + tpr < q.T; t += 2 * tpr) {     // two independent columns in flight per thread
                lse_rows<real, FAST, VE, HT, LOG2OUT>(cta + (int64_t)t * H * hs + j * VE, hs, H, Qall + t * rowElems + j * VE);
                lse_rows<real, FAST, VE, HT, LOG2OUT>(cta + (int64_t)(t + tpr) * H * hs + j * VE, hs, H,
                                             Qall + (t + tpr) * rowElems + j * VE);
            }
            for (; t < q.T; t += tpr)
                lse_rows<real, FAST, VE, HT, LOG2OUT>(cta + (int64_t)t * H * hs + j * VE, hs, H, Qall + t * rowElems + j * VE);
        }
    } else {
        for (int i = tid; i < q.T * nvec; i += nth) {
            const int t = i / nvec, j = i - t * nvec;
            lse_rows<real, FAST, VE, HT, LOG2OUT>(cta + (int64_t)t * H * hs + j * VE, hs, H, Qall + t * rowElems + j * VE);
        }
    }
}

template <typename real, bool FAST, int VE, int HT>
__device__ __forceinline__ void grad_rows(const real *src, real *dst, int64_t hs, int H, const real *f) {
    bool any = false;
#pragma unroll
    for (int k = 0; k < VE; ++k) any |= (f[k] != (real)0);
    if (HT > 0) {
        VecT<real, VE> x[HT > 0 ? HT : 1];
        if (any) {
#pragma unroll
            for (int h = 0; h < (HT > 0 ? HT : 1); ++h) x[h] = ld_cs<real, VE>(src + h * hs);
        }
#pragma unroll
        for (int h = 0; h < (HT > 0 ? HT : 1); ++h) {
            VecT<real, VE> o;
#pragma unroll
            for (int k = 0; k < VE; ++k) o.v[k] = (f[k] == (real)0) ? (real)0 : ex<FAST>(x[h].v[k]) * f[k];
            st_cs<real, VE>(dst + h * hs, o);
        }
    } else {
        for (int h = 0; h < H; ++h) {
            VecT<real, VE> x = ld_cs<real, VE>(src + h * hs);
            VecT<real, VE> o;
#pragma unroll
            for (int k = 0; k < VE; ++k) o.v[k] = (f[k] == (real)0) ? (real)0 : ex<FAST>(x.v[k]) * f[k];
            st_cs<real, VE>(dst + h * hs, o);
        }
    }
}

template <typename real, bool FAST, int VE, int HT>
__device__ __forceinline__ void phase_grad(const Geo &q, const real *__restrict__ lp, const real *Fs,
                                           real *__restrict__ grad, int b0, int Gv, int pitch = 0) {
    const int H = HT > 0 ? HT : q.H;
    const int rowElems = pitch > 0 ? pitch : q.G * q.C;
    const int nvec = (Gv * q.C + VE - 1) / VE;
    const int64_t hs = (int64_t)q.N * q.C;
    const int tid = threadIdx.x, nth = blockDim.x;
    const int64_t cta = (int64_t)b0 * q.C;
    if (nvec <= nth) {
        const int tpr = nth / nvec;
        const int t0 = tid / nvec, j = tid - t0 * nvec;
        if (t0 < tpr)
            for (int t = t0; t < q.T; t += tpr) {
                const int64_t off = cta + (int64_t)t * H * hs + j * VE;
                grad_rows<real, FAST, VE, HT>(lp + off, grad + off, hs, H, Fs + t * rowElems + j * VE);
            }
    } else {
        for (int i = tid; i < q.T * nvec; i += nth) {
            const int t = i / nvec, j = i - t * nvec;
            const int64_t off = cta + (int64_t)t * H * hs + j * VE;
            grad_rows<real, FAST, VE, HT>(lp + off, grad + off, hs, H, Fs + t * rowElems + j * VE);
        }
    }
}

template <typename real, bool FAST, int MODE, int HT>
__global__ void ctc2d_dp_kernel(Geo q, const real *__restrict__ lp, const int64_t *__restrict__ tg,
                                const int64_t *__restrict__ il, const int64_t *__restrict__ tl,
                                const real *__restrict__ grad_out, int64_t go_stride,
                                real *__restrict__ nll_out, real *__restrict__ fac_out, real *__restrict__ grad) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const real NINF = Lim<real>::ninf();
    constexpr int V16 = 16 / (int)sizeof(real);
    const int tid = threadIdx.x, nth = blockDim.x;
    const int b0 = blockIdx.x * q.G;
    const int Gv = min(q.G, q.N - b0);
    const int rowElems = q.G * q.C;
    const int rowStates = q.G * q.SS;
    real *Qall = reinterpret_cast<real *>(smem_raw);            // [T][G*C]
    real *acc = Qall + q.T * rowElems;                           // [T][G*C]  sum of exp(R+Rb+nll), then factor
    real *Ra = acc + q.T * rowElems;                             // [T][G*SS]
    real *As = Ra + q.T * rowStates;                             // [2][G*SS]
    real *fin = As + 2 * rowStates;                              // [2G] final states, then [G] nll
    unsigned char *pres = reinterpret_cast<unsigned char *>(fin + 3 * q.G);  // [T][G*C]

    const StateCtx c = make_ctx(q, b0, Gv, tg, il, tl);
    for (int i = tid; i < q.T * rowElems; i += nth) { acc[i] = 0; pres[i] = 0; }
    if (tid < 2 * q.G) fin[tid] = NINF;

    if (q.vec > 1) phase_q<real, FAST, V16, HT>(q, lp, Qall, b0, Gv);
    else phase_q<real, FAST, 1, HT>(q, lp, Qall, b0, Gv);
    __syncthreads();

    const int gc = c.g * q.C + c.cur;
    // ---- forward sweep (same recurrence as ctc2d_alpha_kernel), one barrier per column
    real R = NINF;
    {
        real *ra = Ra + tid;
        const real *qp = Qall + gc;
        for (int t = 0; t < q.T; ++t) {
            if (c.active) {
                if (t == 0) R = (c.s == 0 || (c.s == 1 && c.L > 0)) ? (real)0 : NINF;
                else if (t < c.Tb && c.in_range) {
                    const real *a = As + ((t - 1) & 1) * rowStates + tid;
                    R = lse3<FAST>(a[0], c.s > 0 ? a[-1] : NINF, c.skip_fwd ? a[-2] : NINF);
                } else R = NINF;
                *ra = R;
                const real a = R + *qp;
                As[(t & 1) * rowStates + tid] = a;
                if (t == c.Tb - 1) {
                    if (c.s == 2 * c.L) fin[2 * c.g] = a;
                    else if (c.s == 2 * c.L - 1) fin[2 * c.g + 1] = a;
                }
            }
            ra += rowStates;
            qp += rowElems;
            __syncthreads();
        }
    }
    real *nlls = fin + 2 * q.G;
    if (c.active && c.s == 0) {
        const real v = -lse2<FAST>(fin[2 * c.g], fin[2 * c.g + 1]);
        nlls[c.g] = v;
        if (MODE != MODE_GRAD) nll_out[c.b] = v;
    }
    __syncthreads();
    const real my_nll = c.active ? nlls[c.g] : (real)0;

    // ---- backward sweep (K2 :283-366) fused with K3's per-class collection (:460-497)
    {
        real Rb = NINF;
        const real *ra = Ra + (q.T - 1) * rowStates + tid;
        int o = (q.T - 1) * rowElems + gc;
        for (int t = q.T - 1; t >= 0; --t) {
            if (c.active) {
                if (t == c.Tb - 1) {
                    Rb = (c.s == 2 * c.L || (c.L > 0 && c.s == 2 * c.L - 1)) ? (real)0 : NINF;
                } else if (t < c.Tb - 1 && c.in_range) {
                    const real *bq = As + ((t + 1) & 1) * rowStates + tid;
                    Rb = lse3<FAST>(bq[0], c.s < 2 * c.L ? bq[1] : NINF, c.skip_bwd ? bq[2] : NINF);
                } else Rb = NINF;
                As[(t & 1) * rowStates + tid] = Rb + Qall[o];
                if (c.in_range && t < c.Tb) {
                    const real v = *ra + Rb;
                    if (v != NINF) {
                        pres[o] = 1;
                        atomicAdd(acc + o, ex<FAST>(v + my_nll));
                    }
                }
            }
            ra -= rowStates;
            o -= rowElems;
            __syncthreads();
        }
    }

    // ---- factor: (1 - acc) [* go] where the class is present and t < Tb, else 0 (K3 :501-515)
    for (int e = tid; e < Gv * q.C; e += nth) {
        const int g = e / q.C;
        const int cc = e - g * q.C;
        const int64_t Tb = il[b0 + g];
        const real gs = (MODE == MODE_GRAD) ? grad_out[(int64_t)(b0 + g) * go_stride] : (real)1;
        real *fo = (MODE != MODE_GRAD) ? fac_out + (int64_t)(b0 + g) * q.C + cc : nullptr;
        const bool dead = (MODE == MODE_FAC_STD) && q.zero_inf && (nlls[g] == -NINF);
        for (int t = 0; t < q.T; ++t) {
            const int o = t * rowElems + e;
            real f = 0;
            if (MODE == MODE_FAC_STD) {
                // aten ctc_loss backward: (exp(lp) - exp(lcab + nll - lp)) * gr for EVERY class, t < Tb
                if (t < Tb && !dead) f = (real)1 - acc[o];
            } else if (pres[o] && t < Tb) f = ((real)1 - acc[o]) * gs;
            if (MODE != MODE_GRAD) fo[(int64_t)t * q.N * q.C] = f;
            else acc[o] = f;
        }
    }
    if (MODE == MODE_GRAD) {
        __syncthreads();
        if (q.vec > 1) phase_grad<real, FAST, V16, HT>(q, lp, acc, grad, b0, Gv);
        else phase_grad<real, FAST, 1, HT>(q, lp, acc, grad, b0, Gv);
    }
}

// ------------------------------------------------------------------------------------------------
// Warp-per-sample DP kernel (fp32, fast math), third revision.  Same phases as ctc2d_dp_kernel, but:
//   * the two sweeps of a sample run inside ONE warp, states in registers (lane L holds states [L*NS, L*NS+NS)),
//     neighbours by warp shuffle, no block barrier inside the 2*T steps (the block version stalls on its barriers);
//   * NS is chosen PER SAMPLE from its target length (2L+1 <= 32 -> one state per lane), so short targets do a third
//     of the work of the padded S = 32 layout;
//   * everything is in log2 units (Q2 = log2(e) * Q): no FMUL around the MUFUs, and the log-sum-exp of three terms
//     costs two ex2 + one lg2 (the largest term contributes exactly 1);
//   * the per-class sums reuse the Q row they correspond to (dead once the backward sweep has passed it) and a bit
//     mask records "class present", so a sample needs T*C + T*(2S+1) floats of shared memory: 16 warps per SM.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float lse3_l2(float a, float b, float c) {
    const float t1 = fmaxf(a, b), t0 = fminf(a, b);
    const float m = fmaxf(t1, c), x1 = fminf(t1, c);
    const float ms = (m == -INFINITY) ? 0.f : m;
    return m + lg2_ftz(1.f + ex2_ftz(x1 - ms) + ex2_ftz(t0 - ms));
}
__device__ __forceinline__ float lse2_l2(float a, float b) {
    const float m = fmaxf(a, b), x = fminf(a, b);
    const float ms = (m == -INFINITY) ? 0.f : m;
    return m + lg2_ftz(1.f + ex2_ftz(x - ms));
}

struct WarpDpCtx {
    const Geo *q;
    const int64_t *row;       // targets of this sample
    int64_t Tb, L;
    float *Qg;                // Q2 rows of this sample: Qg[t * rowElems + c]; later the per-class sums
    float *Rag;               // [T][SS]
    unsigned *maskg;          // [T][MW] class-present bits
    int rowElems, MW;
};

template <int NS, int MODE>
__device__ __forceinline__ float warp_sweeps(const WarpDpCtx &w, int lane) {
    const Geo &q = *w.q;
    const float NINF = -INFINITY;
    const int SS = q.SS;
    const int64_t Tb = w.Tb, L = w.L;
    int cur[NS];
    bool in[NS], skf[NS], skb[NS];
#pragma unroll
    for (int k = 0; k < NS; ++k) {
        const int s = lane * NS + k;
        cur[k] = q.blank; in[k] = skf[k] = skb[k] = false;
        if (s < SS && s < 2 * L + 1) {
            in[k] = L > 0;
            if (s & 1) {
                const int64_t me = w.row[(int64_t)(s >> 1) * q.tg_ss];
                cur[k] = clampi(me, q.C);
                if (s > 1) skf[k] = w.row[(int64_t)((s - 2) >> 1) * q.tg_ss] != me;
                if (s < 2 * L - 1) skb[k] = w.row[(int64_t)((s + 2) >> 1) * q.tg_ss] != me;
            }
        }
    }
    // ---------------- forward sweep
    float R[NS], a[NS];
    float f0 = NINF, f1 = NINF;
#pragma unroll 1
    for (int t = 0; t < q.T; ++t) {
        if (t == 0) {
#pragma unroll
            for (int k = 0; k < NS; ++k) {
                const int s = lane * NS + k;
                R[k] = (s == 0 || (s == 1 && L > 0)) ? 0.f : NINF;
            }
        } else {
            float up1 = __shfl_up_sync(0xffffffffu, a[NS - 1], 1);
            float up2 = NS >= 2 ? __shfl_up_sync(0xffffffffu, a[NS >= 2 ? NS - 2 : 0], 1) : __shfl_up_sync(0xffffffffu, a[0], 2);
            if (lane == 0) up1 = up2 = NINF;
            if (NS == 1 && lane == 1) up2 = NINF;
            float Rn[NS];
#pragma unroll
            for (int k = 0; k < NS; ++k) {
                const float am1 = k >= 1 ? a[k >= 1 ? k - 1 : 0] : up1;
                const float am2 = k >= 2 ? a[k >= 2 ? k - 2 : 0] : (k == 1 ? up1 : up2);
                const float v = lse3_l2(a[k], am1, skf[k] ? am2 : NINF);
                Rn[k] = (t < Tb && in[k]) ? v : NINF;
            }
#pragma unroll
            for (int k = 0; k < NS; ++k) R[k] = Rn[k];
        }
        const float *Qt = w.Qg + t * w.rowElems;
#pragma unroll
        for (int k = 0; k < NS; ++k) {
            const int s = lane * NS + k;
            if (s < SS) w.Rag[t * SS + s] = R[k];
            a[k] = R[k] + Qt[cur[k]];
            if (t == Tb - 1) {
                if (s == 2 * L) f0 = a[k];
                else if (s == 2 * L - 1) f1 = a[k];
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        f0 = fmaxf(f0, __shfl_xor_sync(0xffffffffu, f0, o));
        f1 = fmaxf(f1, __shfl_xor_sync(0xffffffffu, f1, o));
    }
    const float nll2 = -lse2_l2(f0, f1);                    // in log2 units
    // ---------------- backward sweep fused with the per-class collection (the Q row becomes the sum row)
    float bq[NS];
#pragma unroll
    for (int k = 0; k < NS; ++k) bq[k] = NINF;
#pragma unroll 1
    for (int t = q.T - 1; t >= 0; --t) {
        float Rb[NS];
        if (t == Tb - 1) {
#pragma unroll
            for (int k = 0; k < NS; ++k) {
                const int s = lane * NS + k;
                Rb[k] = (s == 2 * L || (L > 0 && s == 2 * L - 1)) ? 0.f : NINF;
            }
        } else if (t < Tb - 1) {
            float dn1 = __shfl_down_sync(0xffffffffu, bq[0], 1);
            float dn2 = NS >= 2 ? __shfl_down_sync(0xffffffffu, bq[NS >= 2 ? 1 : 0], 1) : __shfl_down_sync(0xffffffffu, bq[0], 2);
            if (lane == 31) dn1 = dn2 = NINF;
            if (NS == 1 && lane == 30) dn2 = NINF;
#pragma unroll
            for (int k = 0; k < NS; ++k) {
                const int s = lane * NS + k;
                const float bp1 = k + 1 < NS ? bq[k + 1 < NS ? k + 1 : 0] : dn1;
                const float bp2 = k + 2 < NS ? bq[k + 2 < NS ? k + 2 : 0] : (k + 1 < NS ? dn1 : dn2);
                const float v = lse3_l2(bq[k], s < 2 * L ? bp1 : NINF, skb[k] ? bp2 : NINF);
                Rb[k] = in[k] ? v : NINF;
            }
        } else {
#pragma unroll
            for (int k = 0; k < NS; ++k) Rb[k] = NINF;
        }
        float *Qt = w.Qg + t * w.rowElems;
#pragma unroll
        for (int k = 0; k < NS; ++k) bq[k] = Rb[k] + Qt[cur[k]];
        __syncwarp();                                        // every lane has read Q2[t] -> the row may be reused
        if (q.C <= 64) {                                     // common case: two predicated stores, no loop
            if (lane < q.C) Qt[lane] = 0.f;
            if (lane + 32 < q.C) Qt[lane + 32] = 0.f;
            if (lane < w.MW) w.maskg[t * w.MW + lane] = 0u;
        } else {
            for (int cidx = lane; cidx < q.C; cidx += 32) Qt[cidx] = 0.f;
            for (int mw = lane; mw < w.MW; mw += 32) w.maskg[t * w.MW + mw] = 0u;
        }
        __syncwarp();
        if (t < Tb) {
#pragma unroll
            for (int k = 0; k < NS; ++k) {
                const int s = lane * NS + k;
                if (in[k] && s < SS) {
                    const float v = w.Rag[t * SS + s] + Rb[k];
                    if (v != NINF) {
                        atomicOr(w.maskg + t * w.MW + (cur[k] >> 5), 1u << (cur[k] & 31));
                        atomicAdd(Qt + cur[k], ex2_ftz(v + nll2));
                    }
                }
            }
        }
    }
    __syncwarp();
    return nll2 * 0.6931471805599453f;
}

template <int MODE, int NSMAX, int HT>
__global__ void __launch_bounds__(256)
ctc2d_dp_warp_kernel(Geo q, const float *__restrict__ lp, const int64_t *__restrict__ tg,
                     const int64_t *__restrict__ il, const int64_t *__restrict__ tl,
                     const float *__restrict__ grad_out, int64_t go_stride, float *__restrict__ nll_out,
                     float *__restrict__ fac_out, float *__restrict__ grad) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int b0 = blockIdx.x * q.G;
    const int Gv = min(q.G, q.N - b0);
    const int rowElems = q.G * q.C;
    const int SS = q.SS;
    const int MW = (q.C + 31) >> 5;
    float *Qall = reinterpret_cast<float *>(smem_raw);          // [T][G*C]  Q2, then per-class sums, then factors
    float *Ra = Qall + q.T * rowElems;                           // [G][T][SS]
    unsigned *mask = reinterpret_cast<unsigned *>(Ra + (size_t)q.G * q.T * SS);   // [G][T][MW]
    float *nlls = reinterpret_cast<float *>(mask + (size_t)q.G * q.T * MW);       // [G]

    if (q.vec > 1) phase_q<float, true, 4, HT, true>(q, lp, Qall, b0, Gv);
    else phase_q<float, true, 1, HT, true>(q, lp, Qall, b0, Gv);
    __syncthreads();

    const int g = warp;
    if (g < Gv) {
        const int b = b0 + g;
        WarpDpCtx w;
        w.q = &q; w.row = tg + (int64_t)b * q.tg_sn; w.Tb = il[b]; w.L = tl[b];
        w.Qg = Qall + g * q.C; w.Rag = Ra + (size_t)g * q.T * SS; w.maskg = mask + (size_t)g * q.T * MW;
        w.rowElems = rowElems; w.MW = MW;
        int64_t need64 = 2 * w.L + 1;
        if (need64 > SS) need64 = SS;
        if (need64 < 1) need64 = 1;
        const int need = (int)((need64 + 31) >> 5);
        float nll;
        if (NSMAX == 1 || need <= 1) nll = warp_sweeps<1, MODE>(w, lane);
        else if (NSMAX == 2 || need <= 2) nll = warp_sweeps<(NSMAX >= 2 ? 2 : NSMAX), MODE>(w, lane);
        else if (NSMAX == 3 || need <= 3) nll = warp_sweeps<(NSMAX >= 3 ? 3 : NSMAX), MODE>(w, lane);
        else if (NSMAX == 4 || need <= 4) nll = warp_sweeps<(NSMAX >= 4 ? 4 : NSMAX), MODE>(w, lane);
        else if (NSMAX == 8 || need <= 8) nll = warp_sweeps<(NSMAX >= 8 ? 8 : NSMAX), MODE>(w, lane);
        else if (NSMAX == 16 || need <= 16) nll = warp_sweeps<(NSMAX >= 16 ? 16 : NSMAX), MODE>(w, lane);
        else nll = warp_sweeps<NSMAX, MODE>(w, lane);
        if (lane == 0) {
            nlls[g] = nll;
            if (MODE != MODE_GRAD) nll_out[b] = nll;
        }
        // ---- factor: (1 - sum) [* go] where the class is present and t < Tb, else 0 (K3 :501-515)
        const int64_t Tb = w.Tb;
        const float gs = (MODE == MODE_GRAD) ? grad_out[(int64_t)b * go_stride] : 1.f;
        const bool dead = (MODE == MODE_FAC_STD) && q.zero_inf && (nll == INFINITY);
        for (int t = 0; t < q.T; ++t) {
            float *Qt = w.Qg + t * rowElems;
            for (int c = lane; c < q.C; c += 32) {
                float f = 0.f;
                if (MODE == MODE_FAC_STD) {
                    if (t < Tb && !dead) f = 1.f - Qt[c];
                } else if (t < Tb && ((w.maskg[t * MW + (c >> 5)] >> (c & 31)) & 1u)) f = (1.f - Qt[c]) * gs;
                if (MODE != MODE_GRAD) fac_out[((int64_t)t * q.N + b) * q.C + c] = f;
                else Qt[c] = f;
            }
        }
    }
    if (MODE == MODE_GRAD) {
        __syncthreads();
        if (q.vec > 1) phase_grad<float, true, 4, HT>(q, lp, Qall, grad, b0, Gv);
        else phase_grad<float, true, 1, HT>(q, lp, Qall, grad, b0, Gv);
    }
}

// ------------------------------------------------------------------------------------------------
// Warp-per-sample DP kernel, FOURTH revision (round 2; fp32 fast math; modes GRAD and FAC; S <= 32, C <= 64).
// In the third revision every phase ran as one dependent instruction chain.  What changed:
//   * the forward and the backward sweep of a sample run INTERLEAVED in the same warp: two independent dependency chains
//     per iteration, and T+1 instead of 2T chain steps.  The forward chain covers columns 0..m, the backward chain
//     Tb-1..m (m = Tb/2); they meet at column m, where  -nll = LSE_s(R[m,s] + Rb[m,s] + Q[m,l'_s])  (every path crosses
//     exactly one state of column m), so K3's terms  E[t,s] = exp(R + Rb + nll)  can be formed right there and, in the
//     second half of both chains (forward continues to Tb-1 against the stored Rb rows, backward continues to 0 against
//     the stored R rows), as soon as a step is computed;
//   * only Tb-1 rows of 32*NS floats are stored per sample, and NS is the sample's own ceil((2L+1)/32): the rows live in a
//     pool of G slots per CTA (a sample with long targets takes 2-3 slots; if the CTA's samples need more than G, the
//     warps go in rounds).  Shared memory per CTA drops from 107 KB to 72 KB -> 3 CTAs (24 sample-warps) per SM;
//   * the Q operand of the NEXT step and the stored row it will need are loaded one iteration ahead;
//   * K3's per-class collection is TRANSPOSED: the sweeps only overwrite the consumed row with E[t,s] (one store per
//     state and step, +2^-60 where the state is finite so that "class present" <=> sum > 0); afterwards lane = COLUMN t
//     adds up the blank states and each label state of its column into the (dead) Q row -- ~100 instructions per sample
//     for all 32 columns instead of ~50 per column (16-way same-address atomics on the blank, a CAS loop per label);
//   * phase Q for H = 8 is a straight-line max / fma / ex2 / add sequence (log2 domain); the factor pass has no divisions.
// ------------------------------------------------------------------------------------------------
// log2-domain LSE of three terms with a short dependency chain: max3 -> sub -> ex2 -> add -> lg2 -> add.  The floor on the
// maximum keeps (-inf) - (-inf) from producing NaN: all terms -inf -> 0 + 0 + 0 -> lg2(0) = -inf.
__device__ __forceinline__ float lse3_fast(float a, float b, float c) {
    const float m = fmaxf(fmaxf(a, b), fmaxf(c, -1e30f));
    return m + lg2_ftz(ex2_ftz(a - m) + ex2_ftz(b - m) + ex2_ftz(c - m));
}

#ifndef MR_DP4_PREFETCH
#define MR_DP4_PREFETCH 1
#endif
constexpr bool kDp4Prefetch = MR_DP4_PREFETCH != 0;

struct Dp4Ctx {
    const Geo *q;
    const int64_t *row;       // targets of this sample
    int Tb, L;
    float *Qg;                // Q2 rows of this sample: Qg[t * pitch + c]; later the per-class sums / factors
    float *Rst;               // [T][32*NS + 1] stored sweep rows of this sample, then E[t][s]
    const int *raw;           // [32] the sample's targets (shared memory copy, saturated to int)
    int pitch;
};

// LSE over 8 heights of one 4-wide vector column, result in log2 units.
// LSE over 8 heights of one 4-wide vector column (already in registers), result in log2 units.
__device__ __forceinline__ void lse8_l2(const float4 *x, float *dst) {
    float out[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = k == 0 ? x[u].x : (k == 1 ? x[u].y : (k == 2 ? x[u].z : x[u].w));
        const float m = fmaxf(fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3])), fmaxf(fmaxf(v[4], v[5]), fmaxf(v[6], v[7])));
        const float m2 = m * 1.4426950408889634f;
        const float neg = (m == -INFINITY) ? 0.f : -m2;
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u += 2) {
            s0 += ex2_ftz(fmaf(v[u], 1.4426950408889634f, neg));
            s1 += ex2_ftz(fmaf(v[u + 1], 1.4426950408889634f, neg));
        }
        out[k] = m2 + lg2_ftz(s0 + s1);                       // m = -inf: -inf + lg2(0) = -inf
    }
    *reinterpret_cast<float4 *>(dst) = make_float4(out[0], out[1], out[2], out[3]);
}
template <typename HS>      // HS = int when 8 * N * C fits 31 bits (one IMAD.WIDE per row address), else int64_t
__device__ __forceinline__ void load_rows8(const float *base, HS hs, float4 *x) {
#pragma unroll
    for (int u = 0; u < 8; ++u) x[u] = __ldg(reinterpret_cast<const float4 *>(base + u * hs));
}
template <typename HS>
__device__ __forceinline__ void lse_rows8_l2(const float *base, HS hs, float *dst) {
    float4 x[8];
    load_rows8<HS>(base, hs, x);
    lse8_l2(x, dst);
}

template <typename HS, bool PREFETCH>
__device__ __forceinline__ void phase_q8_l2_impl(const Geo &q, const float *__restrict__ lp, float *Qall, int b0, int Gv, int pitch) {
    const int nvec = (Gv * q.C) >> 2;                        // callers guarantee (Gv*C) % 4 == 0 on this path
    const HS hs = (HS)((int64_t)q.N * q.C);
    const int tid = threadIdx.x, nth = blockDim.x;
    const float *cta = lp + (int64_t)b0 * q.C;
    if (nvec <= nth) {
        const int tpr = nth / nvec;
        const int t0 = tid / nvec, j = tid - t0 * nvec;
        if (t0 < tpr) {
            const float *src = cta + (int64_t)t0 * 8 * (int64_t)hs + j * 4;
            float *dst = Qall + t0 * pitch + j * 4;
            const int64_t sstep = (int64_t)tpr * 8 * (int64_t)hs;
            if (PREFETCH) {
                // the loads of the NEXT column are in flight while this one is reduced (32 more registers)
                float4 xa[8], xb[8];
                load_rows8<HS>(src, hs, xa);
                int t = t0;
                for (; t + tpr < q.T; t += 2 * tpr) {
                    load_rows8<HS>(src + sstep, hs, xb);
                    lse8_l2(xa, dst);
                    if (t + 2 * tpr < q.T) load_rows8<HS>(src + 2 * sstep, hs, xa);
                    lse8_l2(xb, dst + tpr * pitch);
                    src += 2 * sstep; dst += 2 * tpr * pitch;
                }
                if (t < q.T) lse8_l2(xa, dst);
            } else {
                for (int t = t0; t < q.T; t += tpr, src += sstep, dst += tpr * pitch) lse_rows8_l2<HS>(src, hs, dst);
            }
        }
    } else {
        for (int i = tid; i < q.T * nvec; i += nth) {
            const int t = i / nvec, j = i - t * nvec;
            lse_rows8_l2<HS>(cta + (int64_t)t * 8 * (int64_t)hs + j * 4, hs, Qall + t * pitch + j * 4);
        }
    }
}
__device__ __forceinline__ void phase_q8_l2(const Geo &q, const float *__restrict__ lp, float *Qall, int b0, int Gv, int pitch) {
    if ((int64_t)q.N * q.C < (1 << 27)) phase_q8_l2_impl<int, kDp4Prefetch>(q, lp, Qall, b0, Gv, pitch);
    else phase_q8_l2_impl<int64_t, false>(q, lp, Qall, b0, Gv, pitch);
}

// COMPACT: the Q rows hold one column per entry of the sample's own class list (0 = blank, 1 + j = label j) instead of
// one per class of the alphabet (large-alphabet kernel below).
template <int NS, bool COMPACT = false>
__device__ __forceinline__ float warp_sweeps4(const Dp4Ctx &w, int lane) {
    const Geo &q = *w.q;
    const float NINF = -INFINITY;
    const int SS = q.SS;
    const int Tb = w.Tb, L = w.L;
    constexpr int P = 32 * NS + 1;                            // odd row pitch: the transposed pass reads columns
    int cur[NS];
    bool in[NS], skf[NS], skb[NS], succ1[NS];
#pragma unroll
    for (int k = 0; k < NS; ++k) {
        const int s = lane * NS + k;
        cur[k] = COMPACT ? 0 : q.blank; in[k] = skf[k] = skb[k] = false;
        succ1[k] = s < 2 * L;
        if (s < SS && s < 2 * L + 1) {
            in[k] = L > 0;
            if (s & 1) {
                // w.raw[j] = target j as stored (low 32 bits of the int64; the repeat tests of K1/K2 compare labels)
                const int me = w.raw[s >> 1];
                cur[k] = COMPACT ? 1 + (s >> 1) : (me < 0 ? 0 : (me >= q.C ? q.C - 1 : me));
                if (s > 1) skf[k] = w.raw[(s - 2) >> 1] != me;
                if (s < 2 * L - 1) skb[k] = w.raw[(s + 2) >> 1] != me;
            }
        }
    }
    if (Tb < 1) return INFINITY;
    const int m = Tb >> 1;
    const float *Qg = w.Qg;
    const int re = w.pitch;
    float *Rl = w.Rst + lane * NS;                            // this lane's states inside a stored row

    float af[NS], bq[NS], Rf[NS], Rb[NS];
#pragma unroll
    for (int k = 0; k < NS; ++k) af[k] = bq[k] = Rf[k] = Rb[k] = NINF;

    // one forward step: R[t] from A[t-1] (held in af), then A[t] = R[t] + Q[t]
    auto fwd_step = [&](int t, const float *qv) {
        if (t == 0) {
#pragma unroll
            for (int k = 0; k < NS; ++k) {
                const int s = lane * NS + k;
                Rf[k] = (s == 0 || (s == 1 && L > 0)) ? 0.f : NINF;
            }
        } else {
            float up1 = __shfl_up_sync(0xffffffffu, af[NS - 1], 1);
            float up2 = NS >= 2 ? __shfl_up_sync(0xffffffffu, af[NS >= 2 ? NS - 2 : 0], 1) : __shfl_up_sync(0xffffffffu, af[0], 2);
            if (lane == 0) up1 = up2 = NINF;
            if (NS == 1 && lane == 1) up2 = NINF;
            float Rn[NS];
#pragma unroll
            for (int k = 0; k < NS; ++k) {
                const float am1 = k >= 1 ? af[k >= 1 ? k - 1 : 0] : up1;
                const float am2 = k >= 2 ? af[k >= 2 ? k - 2 : 0] : (k == 1 ? up1 : up2);
                const float v = lse3_fast(af[k], am1, skf[k] ? am2 : NINF);
                Rn[k] = in[k] ? v : NINF;
            }
#pragma unroll
            for (int k = 0; k < NS; ++k) Rf[k] = Rn[k];
        }
#pragma unroll
        for (int k = 0; k < NS; ++k) af[k] = Rf[k] + qv[k];
    };
    // one backward step: Rb[t] from B[t+1] (held in bq), then B[t] = Rb[t] + Q[t]
    auto bwd_step = [&](int t, const float *qv) {
        if (t == Tb - 1) {
#pragma unroll
            for (int k = 0; k < NS; ++k) {
                const int s = lane * NS + k;
                Rb[k] = (s == 2 * L || (L > 0 && s == 2 * L - 1)) ? 0.f : NINF;
            }
        } else {
            float dn1 = __shfl_down_sync(0xffffffffu, bq[0], 1);
            float dn2 = NS >= 2 ? __shfl_down_sync(0xffffffffu, bq[NS >= 2 ? 1 : 0], 1) : __shfl_down_sync(0xffffffffu, bq[0], 2);
            if (lane == 31) dn1 = dn2 = NINF;
            if (NS == 1 && lane == 30) dn2 = NINF;
            float Rn[NS];
#pragma unroll
            for (int k = 0; k < NS; ++k) {
                const float bp1 = k + 1 < NS ? bq[k + 1 < NS ? k + 1 : 0] : dn1;
                const float bp2 = k + 2 < NS ? bq[k + 2 < NS ? k + 2 : 0] : (k + 1 < NS ? dn1 : dn2);
                const float v = lse3_fast(bq[k], succ1[k] ? bp1 : NINF, skb[k] ? bp2 : NINF);
                Rn[k] = in[k] ? v : NINF;
            }
#pragma unroll
            for (int k = 0; k < NS; ++k) Rb[k] = Rn[k];
        }
#pragma unroll
        for (int k = 0; k < NS; ++k) bq[k] = Rb[k] + qv[k];
    };
    auto load_q = [&](int t, float *qv) {
        const float *Qt = Qg + t * re;
#pragma unroll
        for (int k = 0; k < NS; ++k) qv[k] = Qt[cur[k]];
    };
    // K3's term of column t for this lane's states: E = exp2(R + Rb + nll2) (+ 2^-60: "this state is finite"), else 0
    auto emit = [&](int t, const float *v, float nll2) {
#pragma unroll
        for (int k = 0; k < NS; ++k) {
            const int s = lane * NS + k;
            const bool ok = in[k] && s < SS && v[k] != NINF;
            Rl[t * P + k] = ok ? ex2_ftz(v[k] + nll2) + 0x1p-60f : 0.f;
        }
    };

    // ---------------- phase 1: forward columns 0..m, backward columns Tb-1..m (stored: forward 0..m-1, backward m+1..Tb-1)
    float qf[NS], qb[NS];
    load_q(0, qf);
    load_q(Tb - 1, qb);
    const int nb1 = Tb - m;                                   // backward steps of phase 1 (Tb-1 .. m)
#pragma unroll 1
    for (int i = 0; i <= m; ++i) {
        float qfn[NS], qbn[NS];
        load_q(min(i + 1, Tb - 1), qfn);
        load_q(max(Tb - 2 - i, 0), qbn);
        fwd_step(i, qf);
        if (i < m) {
#pragma unroll
            for (int k = 0; k < NS; ++k) Rl[i * P + k] = Rf[k];
        }
        if (i < nb1) {
            const int tb = Tb - 1 - i;
            bwd_step(tb, qb);
            if (tb > m) {
#pragma unroll
                for (int k = 0; k < NS; ++k) Rl[tb * P + k] = Rb[k];
            }
#pragma unroll
            for (int k = 0; k < NS; ++k) qb[k] = qbn[k];
        }
#pragma unroll
        for (int k = 0; k < NS; ++k) qf[k] = qfn[k];
    }
    // ---------------- meeting column m: -nll2 = LSE2_s( R[m,s] + Rb[m,s] + Q2[m, l'_s] ) = LSE2_s( af[s] + Rb[s] )
    float nll2;
    {
        float mx = NINF;
        float tv[NS];
#pragma unroll
        for (int k = 0; k < NS; ++k) {
            const int s = lane * NS + k;
            tv[k] = (s < SS) ? af[k] + Rb[k] : NINF;
            mx = fmaxf(mx, tv[k]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (mx == NINF) nll2 = INFINITY;
        else {
            float sm = 0.f;
#pragma unroll
            for (int k = 0; k < NS; ++k) sm += ex2_ftz(tv[k] - mx);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sm += __shfl_xor_sync(0xffffffffu, sm, o);
            nll2 = -(mx + lg2_ftz(sm));
        }
        float v[NS];
#pragma unroll
        for (int k = 0; k < NS; ++k) v[k] = Rf[k] + Rb[k];
        emit(m, v, nll2);
    }
    // ---------------- phase 2: forward m+1..Tb-1 against the stored Rb rows, backward m-1..0 against the stored R rows
    const int nf2 = Tb - 1 - m, nb2 = m;
    const int n2 = nf2 > nb2 ? nf2 : nb2;
    float sf[NS], sb[NS];                                     // stored rows for the current iteration
    {
        const int tf = min(m + 1, Tb - 1), tb = max(m - 1, 0);
#pragma unroll
        for (int k = 0; k < NS; ++k) { sf[k] = Rl[tf * P + k]; sb[k] = Rl[tb * P + k]; }
    }
#pragma unroll 1
    for (int j = 0; j < n2; ++j) {
        const int tf = m + 1 + j, tb = m - 1 - j;
        float qfn[NS], qbn[NS], sfn[NS], sbn[NS];
        {
            const int tfn = min(tf + 1, Tb - 1), tbn = max(tb - 1, 0);
            load_q(tfn, qfn);
            load_q(tbn, qbn);
#pragma unroll
            for (int k = 0; k < NS; ++k) { sfn[k] = Rl[tfn * P + k]; sbn[k] = Rl[tbn * P + k]; }
        }
        if (j < nf2) {
            fwd_step(tf, qf);
            float v[NS];
#pragma unroll
            for (int k = 0; k < NS; ++k) v[k] = Rf[k] + sf[k];
            emit(tf, v, nll2);
        }
        if (j < nb2) {
            bwd_step(tb, qb);
            float v[NS];
#pragma unroll
            for (int k = 0; k < NS; ++k) v[k] = sb[k] + Rb[k];
            emit(tb, v, nll2);
        }
#pragma unroll
        for (int k = 0; k < NS; ++k) { qf[k] = qfn[k]; qb[k] = qbn[k]; sf[k] = sfn[k]; sb[k] = sbn[k]; }
    }
    __syncwarp();                                             // E rows complete; every lane is done with the Q rows
    // ---------------- transposed collection: lane = column t.  sums[t][class] (in the dead Q row) = sum of E over the
    // states of that class; the first label of a class stores, later ones add (firstbits from the caller).
    return nll2 * 0.6931471805599453f;
}

// lane = column: per-class sums of E[t][s] into the Q row of column t.  cls[j] = class of label j, firstbits bit j = label j
// is the first label of its class.
template <int NS>
__device__ __forceinline__ void collect_transposed(const Dp4Ctx &w, int lane, const int *cls, unsigned firstbits,
                                                   int blank_slot = -1) {
    constexpr int P = 32 * NS + 1;
    const int L = w.L;
    const int blank = blank_slot >= 0 ? blank_slot : w.q->blank;
    for (int t0 = 0; t0 < w.Tb; t0 += 32) {
        const int t = t0 + lane;
        if (t < w.Tb) {
            const float *Et = w.Rst + t * P;
            float *Qt = w.Qg + t * w.pitch;
            float a0 = 0.f, a1 = 0.f;
            int s = 0;
            for (; s + 2 <= 2 * L; s += 4) { a0 += Et[s]; a1 += Et[s + 2]; }
            if (s <= 2 * L) a0 += Et[s];
            Qt[blank] = a0 + a1;
            for (int j = 0; j < L; ++j) {
                const float e = Et[2 * j + 1];
                float *dst = Qt + cls[j];
                *dst = ((firstbits >> j) & 1u) ? e : *dst + e;
            }
        }
    }
    __syncwarp();
}

template <int MODE, int HT>
__global__ void __launch_bounds__(256, 3)
ctc2d_dp4_kernel(Geo q, const float *__restrict__ lp, const int64_t *__restrict__ tg,
                 const int64_t *__restrict__ il, const int64_t *__restrict__ tl,
                 const float *__restrict__ grad_out, int64_t go_stride, float *__restrict__ nll_out,
                 float *__restrict__ fac_out, float *__restrict__ grad, int pitch) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int b0 = blockIdx.x * q.G;
    const int Gv = min(q.G, q.N - b0);
    float *Qall = reinterpret_cast<float *>(smem_raw);           // [T][pitch]  Q2, then per-class sums, then factors
    float *pool = Qall + q.T * pitch;                             // [max(G,3) slots][T][33]
    const int nslots = q.G > 3 ? q.G : 3;                         // a single sample may need 3 slots (S = 32: 65 states)
    int *meta = reinterpret_cast<int *>(pool + (size_t)nslots * q.T * 33);   // [G] slot, round, ns, Tb, L; [1] rounds
    unsigned *tmask = reinterpret_cast<unsigned *>(meta + 5 * q.G + 1);   // [G][2] classes that occur in the extended target
    int *cls = reinterpret_cast<int *>(tmask + 2 * q.G);          // [G][32] class of label j
    int *raw = cls + 32 * q.G;                                    // [G][32] targets as stored
    for (int i = tid; i < Gv * 32; i += blockDim.x) {            // (S <= 32 on this path)
        const int gg = i >> 5, j = i & 31;
        int64_t v = j < q.S ? tg[(int64_t)(b0 + gg) * q.tg_sn + (int64_t)j * q.tg_ss] : 0;
        raw[i] = v < -2147483647 ? -2147483647 : (v > 2147483647 ? 2147483647 : (int)v);
    }

    if (tid == 0) {                                              // slot / round plan of this CTA's samples
        int used = 0, round = 0;
        for (int g = 0; g < q.G; ++g) {
            int ns = 1, Tb = 0, L = 0;
            if (g < Gv) {
                int64_t L64 = tl[b0 + g], T64 = il[b0 + g];
                if (L64 < 0) L64 = 0;
                if (L64 > q.S) L64 = q.S;
                if (T64 < 0) T64 = 0;
                if (T64 > q.T) T64 = q.T;
                L = (int)L64; Tb = (int)T64;
                ns = (2 * L + 1 + 31) >> 5;
            }
            if (used + ns > nslots) { ++round; used = 0; }
            meta[g] = used; meta[q.G + g] = round; meta[2 * q.G + g] = ns; meta[3 * q.G + g] = Tb; meta[4 * q.G + g] = L;
            used += ns;
        }
        meta[5 * q.G] = round + 1;
    }
    if (HT == 8 && q.vec > 1) phase_q8_l2(q, lp, Qall, b0, Gv, pitch);
    else if (q.vec > 1) phase_q<float, true, 4, HT, true>(q, lp, Qall, b0, Gv, pitch);
    else phase_q<float, true, 1, HT, true>(q, lp, Qall, b0, Gv, pitch);
    __syncthreads();

    const int rounds = meta[5 * q.G];
    const int g = warp;
    for (int r = 0; r < rounds; ++r) {
        if (g < Gv && meta[q.G + g] == r) {
            const int b = b0 + g;
            Dp4Ctx w;
            w.q = &q; w.row = tg + (int64_t)b * q.tg_sn; w.Tb = meta[3 * q.G + g]; w.L = meta[4 * q.G + g];
            w.Qg = Qall + g * q.C; w.Rst = pool + (size_t)meta[g] * q.T * 33; w.pitch = pitch; w.raw = raw + g * 32;
            const int ns = meta[2 * q.G + g];
            // labels of this sample (lane j = label j; S <= 32), the classes that occur, and "first label of its class"
            const int rawc = w.raw[lane];
            const int myc = lane < w.L ? (rawc < 0 ? 0 : (rawc >= q.C ? q.C - 1 : rawc)) : -1 - lane;
            unsigned lo = (lane == 0) ? (q.blank < 32 ? 1u << q.blank : 0u) : 0u;
            unsigned hi = (lane == 0) ? (q.blank >= 32 ? 1u << (q.blank - 32) : 0u) : 0u;
            if (myc >= 0) { if (myc < 32) lo |= 1u << myc; else hi |= 1u << (myc - 32); }
            lo = __reduce_or_sync(0xffffffffu, lo);
            hi = __reduce_or_sync(0xffffffffu, hi);
            const unsigned same = __match_any_sync(0xffffffffu, myc);
            const unsigned firstbits = __ballot_sync(0xffffffffu, myc >= 0 && (__ffs(same) - 1) == lane);
            cls[g * 32 + lane] = myc >= 0 ? myc : 0;
            if (lane == 0) { tmask[2 * g] = lo; tmask[2 * g + 1] = hi; }
            __syncwarp();
            float nll;
            if (ns <= 1) { nll = warp_sweeps4<1>(w, lane); collect_transposed<1>(w, lane, cls + g * 32, firstbits); }
            else if (ns == 2) { nll = warp_sweeps4<2>(w, lane); collect_transposed<2>(w, lane, cls + g * 32, firstbits); }
            else { nll = warp_sweeps4<3>(w, lane); collect_transposed<3>(w, lane, cls + g * 32, firstbits); }
            if (MODE != MODE_GRAD && lane == 0) nll_out[b] = nll;
        }
        if (rounds > 1) __syncthreads();
    }
    __syncthreads();
    // ---- factor: (1 - sum) [* go] where the class is present and t < Tb, else 0 (K3 :501-515).  Thread = fixed vector
    // column of the [Gv*C] row (sample / class bits / lengths are loop invariants), loop over t: no divisions in the loop.
    auto factor_of = [](float sum, float gs) {
        float f = 0.f;
        if (sum > 0.f) {
            f = 1.f - sum;
            if (f == 0.f) f = 0x1p-30f;             // exact cancellation must not read as "class absent" (grad == 0 pattern)
            f *= gs;
        }
        return f;
    };
    const int64_t ostep = (int64_t)q.N * q.C;
    if (q.vec > 1) {
        for (int e4 = tid; e4 < (Gv * q.C) >> 2; e4 += blockDim.x) {
            int tbs[4];
            float gsv[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int e = e4 * 4 + k;
                const int gg = e / q.C, c = e - gg * q.C;
                const bool listed = (c < 32 ? (tmask[2 * gg] >> c) : (tmask[2 * gg + 1] >> (c - 32))) & 1u;
                tbs[k] = listed ? meta[3 * q.G + gg] : 0;
                gsv[k] = (MODE == MODE_GRAD) ? grad_out[(int64_t)(b0 + gg) * go_stride] : 1.f;
            }
            float *col = Qall + e4 * 4;
            float *out = (MODE != MODE_GRAD) ? fac_out + (int64_t)b0 * q.C + e4 * 4 : nullptr;
#pragma unroll 4
            for (int t = 0; t < q.T; ++t) {
                const float4 sv = *reinterpret_cast<const float4 *>(col + t * pitch);
                float4 f;
                f.x = t < tbs[0] ? factor_of(sv.x, gsv[0]) : 0.f;
                f.y = t < tbs[1] ? factor_of(sv.y, gsv[1]) : 0.f;
                f.z = t < tbs[2] ? factor_of(sv.z, gsv[2]) : 0.f;
                f.w = t < tbs[3] ? factor_of(sv.w, gsv[3]) : 0.f;
                if (MODE != MODE_GRAD) *reinterpret_cast<float4 *>(out + t * ostep) = f;
                else *reinterpret_cast<float4 *>(col + t * pitch) = f;
            }
        }
    } else {
        for (int e = tid; e < Gv * q.C; e += blockDim.x) {
            const int gg = e / q.C, c = e - gg * q.C;
            const bool listed = (c < 32 ? (tmask[2 * gg] >> c) : (tmask[2 * gg + 1] >> (c - 32))) & 1u;
            const int Tb = listed ? meta[3 * q.G + gg] : 0;
            const float gs = (MODE == MODE_GRAD) ? grad_out[(int64_t)(b0 + gg) * go_stride] : 1.f;
            float *col = Qall + e;
            float *out = (MODE != MODE_GRAD) ? fac_out + (int64_t)b0 * q.C + e : nullptr;
            for (int t = 0; t < q.T; ++t) {
                const float f = t < Tb ? factor_of(col[t * pitch], gs) : 0.f;
                if (MODE != MODE_GRAD) out[t * ostep] = f;
                else col[t * pitch] = f;
            }
        }
    }
    if (MODE == MODE_GRAD) {
        __syncthreads();
        if (q.vec > 1) phase_grad<float, true, 4, HT>(q, lp, Qall, grad, b0, Gv, pitch);
        else phase_grad<float, true, 1, HT>(q, lp, Qall, grad, b0, Gv, pitch);
    }
}

// ------------------------------------------------------------------------------------------------
// Large alphabets (ChineseCharset: ~5 k classes, concern/charsets.py:65-78) -- the reference's dead "is_large" path, K4
// (:371-424, :557-602), asked the same question.  The dynamic programme only ever touches the classes of the sample's own
// extended target (blank + at most S labels), so nothing of size C needs to live on chip: one WARP per sample gathers
// Q[t][j] = LSE_h lp[t,h,b,class_j] for its <= 33 classes, runs the same interleaved sweeps on those compact rows, and
// scatters the <= 33 non-zero factors (or gradient columns) per time step into rows that it zero-fills itself.
// Shared memory per sample: T * (33 + 33*NS) floats, independent of C.  fp32 fast math, S <= 32.
// ------------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(128)
ctc2d_dpg_kernel(Geo q, const float *__restrict__ lp, const int64_t *__restrict__ tg, const int64_t *__restrict__ il,
                 const int64_t *__restrict__ tl, const float *__restrict__ grad_out, int64_t go_stride,
                 float *__restrict__ nll_out, float *__restrict__ fac_out, float *__restrict__ grad) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * 4 + warp;
    if (b >= q.N) return;
    const size_t per_warp = (size_t)q.T * (33 + 99) + 96;
    float *Qc = reinterpret_cast<float *>(smem_raw) + warp * per_warp;     // [T][33] compact Q2 rows, then sums / factors
    float *Rst = Qc + (size_t)q.T * 33;                                     // [T][33*NS] sweep rows, then E
    int *raw = reinterpret_cast<int *>(Rst + (size_t)q.T * 99);             // [32] targets as stored
    int *slot = raw + 32;                                                   // [32] compact slot that collects label j
    int *clsv = slot + 32;                                                  // [32] class of label j (clamped)
    int64_t L64 = tl[b], T64 = il[b];
    if (L64 < 0) L64 = 0;
    if (L64 > q.S) L64 = q.S;
    if (T64 < 0) T64 = 0;
    if (T64 > q.T) T64 = q.T;
    const int L = (int)L64, Tb = (int)T64;
    {
        const int64_t v = lane < q.S ? tg[(int64_t)b * q.tg_sn + (int64_t)lane * q.tg_ss] : 0;
        const int r = v < -2147483647 ? -2147483647 : (v > 2147483647 ? 2147483647 : (int)v);
        raw[lane] = r;
        const int myc = lane < L ? (r < 0 ? 0 : (r >= q.C ? q.C - 1 : r)) : -1 - lane;
        const unsigned same = __match_any_sync(0xffffffffu, myc);
        slot[lane] = 1 + (__ffs(same) - 1);                                 // first label with the same class collects
        clsv[lane] = myc >= 0 ? myc : 0;
    }
    __syncwarp();
    const unsigned firstbits = __ballot_sync(0xffffffffu, lane < L && slot[lane] == 1 + lane);
    const int64_t hs = (int64_t)q.N * q.C;                                  // stride between heights
    const float *base = lp + (int64_t)b * q.C;
    // ---- Q2[t][j], j = 0 (blank), 1 + label index: gathered columns, log2 units
    for (int j = lane; j <= L; j += 32) {
        const int c = j == 0 ? q.blank : clsv[j - 1];
        const float *p = base + c;
        for (int t = 0; t < q.T; ++t) {
            const float *pt = p + (int64_t)t * q.H * hs;
            float m = -INFINITY;
            for (int h = 0; h < q.H; ++h) m = fmaxf(m, __ldg(pt + h * hs));
            const float m2 = m * 1.4426950408889634f;
            const float neg = (m == -INFINITY) ? 0.f : -m2;
            float sum = 0.f;
            for (int h = 0; h < q.H; ++h) sum += ex2_ftz(fmaf(__ldg(pt + h * hs), 1.4426950408889634f, neg));
            Qc[t * 33 + j] = m2 + lg2_ftz(sum);
        }
    }
    __syncwarp();
    Dp4Ctx w;
    w.q = &q; w.row = nullptr; w.Tb = Tb; w.L = L; w.Qg = Qc; w.Rst = Rst; w.raw = raw; w.pitch = 33;
    const int ns = (2 * L + 1 + 31) >> 5;
    float nll;
    if (ns <= 1) { nll = warp_sweeps4<1, true>(w, lane); collect_transposed<1>(w, lane, slot, firstbits, 0); }
    else if (ns == 2) { nll = warp_sweeps4<2, true>(w, lane); collect_transposed<2>(w, lane, slot, firstbits, 0); }
    else { nll = warp_sweeps4<3, true>(w, lane); collect_transposed<3>(w, lane, slot, firstbits, 0); }
    if (MODE != MODE_GRAD && lane == 0) nll_out[b] = nll;
    // ---- outputs: zero rows, then the columns of the target's classes.  K3 :501-515: (1 - sum) [* go] where present
    const float gs = (MODE == MODE_GRAD) ? grad_out[(int64_t)b * go_stride] : 1.f;
    if (MODE != MODE_GRAD) {
        for (int t = 0; t < q.T; ++t) {
            float *row = fac_out + ((int64_t)t * q.N + b) * q.C;
            for (int c = lane; c < q.C; c += 32) row[c] = 0.f;
        }
    } else {
        for (int r = 0; r < q.T * q.H; ++r) {
            float *row = grad + (int64_t)r * hs + (int64_t)b * q.C;
            for (int c = lane; c < q.C; c += 32) row[c] = 0.f;
        }
    }
    __syncwarp();
    for (int j = lane; j <= L; j += 32) {
        if (j > 0 && !((firstbits >> (j - 1)) & 1u)) continue;              // a later label of an already collected class
        const int c = j == 0 ? q.blank : clsv[j - 1];
        for (int t = 0; t < Tb; ++t) {
            const float sum = Qc[t * 33 + j];
            float f = 0.f;
            if (sum > 0.f) {
                f = 1.f - sum;
                if (f == 0.f) f = 0x1p-30f;
                f *= gs;
            }
            if (MODE != MODE_GRAD) fac_out[((int64_t)t * q.N + b) * q.C + c] = f;
            else if (f != 0.f) {
                const float *pt = base + c + (int64_t)t * q.H * hs;
                float *gt = grad + (int64_t)b * q.C + c + (int64_t)t * q.H * hs;
                for (int h = 0; h < q.H; ++h) gt[h * hs] = ex2_ftz(__ldg(pt + h * hs) * 1.4426950408889634f) * f;
            }
        }
    }
}

// Training backward: grad[t,h,b,c] = exp(lp) * gfac[t,b,c] * go[b].  Pure streaming.  blockIdx.y = t, thread = one
// 16-byte vector column of the [N*C] row; the factor is formed once and reused for the H rows.
template <bool FAST, int VE, int HT>
__global__ void __launch_bounds__(256)
ctc2d_apply_kernel(const float *__restrict__ lp, const float *__restrict__ fac, const float *__restrict__ go,
                   int64_t go_stride, int T, int Hrt, int N, int C, float *__restrict__ grad) {
    const int H = HT > 0 ? HT : Hrt;
    const int64_t row = (int64_t)N * C;
    const int64_t nvec_row = row / VE;
    const int t = blockIdx.y;
    for (int64_t jv = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; jv < nvec_row; jv += (int64_t)gridDim.x * blockDim.x) {
        const int64_t j = jv * VE;
        VecT<float, VE> fv = ld_nc<float, VE>(fac + (int64_t)t * row + j);
        float f[VE];
#pragma unroll
        for (int k = 0; k < VE; ++k) {
            const int b = (int)((j + k) / C);
            f[k] = fv.v[k] * __ldg(go + (int64_t)b * go_stride);
        }
        const int64_t off = (int64_t)t * H * row + j;
        grad_rows<float, FAST, VE, HT>(lp + off, grad + off, row, H, f);
    }
}

// ---- 1D CTC helpers: one warp per (t, b) row of C classes ----
__global__ void rows_log_softmax_kernel(const float *__restrict__ x, int64_t rows, int C, float *__restrict__ out) {
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    const float *p = x + r * C;
    float m = -INFINITY;
    for (int c = lane; c < C; c += 32) m = fmaxf(m, p[c]);
    for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) sum += expf(p[c] - m);
    for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
    const float lse = m + logf(sum);
    for (int c = lane; c < C; c += 32) out[r * C + c] = p[c] - lse;
}

// grad_logits[r,c] = scale[b] * (g - p * sum_c g),  g = p * fac,  p = exp(lp)   (CTC grad folded through log_softmax)
__global__ void ctc1d_grad_rows_kernel(const float *__restrict__ lp, const float *__restrict__ fac,
                                       const float *__restrict__ scale, int64_t rows, int N, int C,
                                       float *__restrict__ grad) {
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    const int b = (int)(r % N);
    const float sc = scale[b];
    const float *l = lp + r * C, *f = fac + r * C;
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) sum += expf(l[c]) * f[c];
    for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
    for (int c = lane; c < C; c += 32) {
        const float p = expf(l[c]);
        grad[r * C + c] = sc * (p * f[c] - p * sum);
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int check_common(const void *lp, const void *tg, const void *il, const void *tl, int64_t T, int64_t H, int64_t N,
                 int64_t C, int64_t S, int64_t blank) {
    if (T < 0 || H < 0 || N < 0 || C <= 0 || S < 0) return MR_ERR_BAD_SHAPE;
    if (blank < 0 || blank >= C) return MR_ERR_BLANK_RANGE;
    if (2 * S + 1 > 1024) return MR_ERR_TARGET_TOO_LONG;
    if (T > (1 << 24) || H > (1 << 20) || C > (1 << 24) || N > (1LL << 31) - 1) return MR_ERR_BAD_SHAPE;
    if (N > 0 && T > 0 && H > 0 && (!lp || !tg || !il || !tl)) return MR_ERR_NULL_POINTER;
    return MR_OK;
}

template <typename real>
int pick_vec(const void *p, int64_t N, int64_t C, int G) {
    const int ve = 16 / (int)sizeof(real);
    if (((uintptr_t)p % 16) == 0 && (N * C) % ve == 0 && ((int64_t)G * C) % ve == 0) return ve;
    return 1;
}

int smem_limit() {
    static int lim = -1;
    if (lim < 0) {
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
            v = 48 * 1024;
        lim = v;
    }
    return lim;
}

template <typename real, bool FAST>
int launch_alpha(const real *lp, const int64_t *tg, const int64_t *il, const int64_t *tl, int64_t T, int64_t H,
                 int64_t N, int64_t C, int64_t S, int64_t tg_sn, int64_t tg_ss, int64_t blank, real *nll, real *la,
                 cudaStream_t st) {
    Geo q;
    q.zero_inf = 0;
    q.T = (int)T; q.H = (int)H; q.N = (int)N; q.C = (int)C; q.S = (int)S; q.SS = (int)(2 * S + 1);
    q.blank = (int)blank; q.tg_sn = tg_sn; q.tg_ss = tg_ss;
    int G = 288 / q.SS;
    if (G < 1) G = 1;
    if (G > 8) G = 8;
    const size_t small = sizeof(real) * ((size_t)G * C + (size_t)G * q.SS + 2 * G);
    // staged path: kStages slabs of [H][G*C]; shrink G until it fits (<= ~56 KB keeps 4 CTAs/SM)
    bool staged = false;
    int Gs = G;
    for (; Gs >= 1; --Gs) {
        const size_t need = sizeof(real) * (size_t)kStages * H * Gs * C + sizeof(real) * ((size_t)Gs * C + (size_t)Gs * q.SS + 2 * Gs);
        if (need <= (size_t)56 * 1024 || (Gs == 1 && need <= (size_t)smem_limit())) { staged = true; break; }
    }
    size_t smem;
    if (staged) {
        G = Gs;
        smem = sizeof(real) * (size_t)kStages * H * G * C + sizeof(real) * ((size_t)G * C + (size_t)G * q.SS + 2 * G);
    } else {
        // large alphabets: shrink the CTA's sample group until the un-staged plan fits
        auto small_need = [&](int g) { return sizeof(real) * ((size_t)g * C + (size_t)g * q.SS + 2 * g); };
        while (G > 1 && small_need(G) > (size_t)smem_limit()) --G;
        smem = small_need(G);
        if (smem > (size_t)smem_limit()) return MR_ERR_UNSUPPORTED;
    }
    q.G = G;
    q.vec = pick_vec<real>(lp, N, C, G);
    const int threads = (int)round_up((int64_t)G * q.SS, 32);
    const int grid = (int)ceil_div(N, G);
    auto kern = staged ? (H == 8 ? ctc2d_alpha_kernel<real, FAST, true, 8> : ctc2d_alpha_kernel<real, FAST, true, 0>)
                       : ctc2d_alpha_kernel<real, FAST, false, 0>;
    if (smem > 48 * 1024)
        MR_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "ctc2d_alpha attr");
    kern<<<grid, threads, smem, st>>>(q, lp, tg, il, tl, nll, la);
    return check_launch("ctc2d_alpha_kernel");
}

template <int MODE, int NSMAX>
int launch_dp_warp_ns(Geo q, const float *lp, const int64_t *tg, const int64_t *il, const int64_t *tl, const float *go,
                      int64_t go_stride, float *nll, float *fac, float *grad, size_t smem, cudaStream_t st) {
    auto kern = (q.H == 8) ? ctc2d_dp_warp_kernel<MODE, NSMAX, 8> : ctc2d_dp_warp_kernel<MODE, NSMAX, 0>;
    if (smem > 48 * 1024)
        MR_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "ctc2d_dp_warp attr");
    kern<<<(unsigned)ceil_div(q.N, q.G), 256, smem, st>>>(q, lp, tg, il, tl, go, go_stride, nll, fac, grad);
    return check_launch("ctc2d_dp_warp_kernel");
}

// returns MR_ERR_UNSUPPORTED when the warp kernel's shared-memory plan does not fit (caller falls back)
template <int MODE>
int launch_dp_warp(Geo q, const float *lp, const int64_t *tg, const int64_t *il, const int64_t *tl, const float *go,
                   int64_t go_stride, float *nll, float *fac, float *grad, cudaStream_t st) {
    const int need_ns = (q.SS + 31) / 32;
    const int opts[] = {1, 2, 3, 4, 8, 16, 32};
    int NS = 0;
    for (int o : opts) if (o >= need_ns) { NS = o; break; }
    if (!NS) return MR_ERR_UNSUPPORTED;
    int G = 8;                                               // one warp per sample, 8 samples per CTA
    auto need = [&](int g) {
        return sizeof(float) * ((size_t)q.T * g * q.C + (size_t)g * q.T * q.SS + g) +
               sizeof(unsigned) * (size_t)g * q.T * ((q.C + 31) / 32) + 16;
    };
    while (G > 1 && need(G) > (size_t)110 * 1024) --G;
    const size_t smem = need(G);
    if (smem > (size_t)smem_limit()) return MR_ERR_UNSUPPORTED;
    q.G = G;
    q.vec = pick_vec<float>(lp, q.N, q.C, G);
    if (MODE == MODE_GRAD && ((uintptr_t)grad % 16) != 0) q.vec = 1;
#define MR_NS(NSV) case NSV: return launch_dp_warp_ns<MODE, NSV>(q, lp, tg, il, tl, go, go_stride, nll, fac, grad, smem, st)
    switch (NS) { MR_NS(1); MR_NS(2); MR_NS(3); MR_NS(4); MR_NS(8); MR_NS(16); MR_NS(32); }
#undef MR_NS
    return MR_ERR_UNSUPPORTED;
}

// Fourth-revision warp DP kernel (ctc2d_dp4_kernel): fp32 fast math, modes GRAD / FAC, S <= 32, C <= 64.
// Returns MR_ERR_UNSUPPORTED otherwise (callers fall back to the v3 / block kernels).
template <int MODE>
int launch_dp4(Geo q, const float *lp, const int64_t *tg, const int64_t *il, const int64_t *tl, const float *go,
               int64_t go_stride, float *nll, float *fac, float *grad, cudaStream_t st) {
    if (MODE == MODE_FAC_STD || q.S > 32 || q.C > 64) return MR_ERR_UNSUPPORTED;
    // row pitch of the Q / sums rows: = 4 (mod 8) floats, so that the transposed pass (lane = column t, same class) hits
    // 8 different banks, and a multiple of 4 whenever the rows are accessed as float4
    auto pitch_of = [&](int g) { int p = g * q.C; while (p % 8 != 4) ++p; return p; };
    auto need = [&](int g) {
        return sizeof(float) * ((size_t)q.T * pitch_of(g) + (size_t)(g > 3 ? g : 3) * q.T * 33) + sizeof(int) * (size_t)(7 * g + 1 + 64 * g) + 16;
    };
    int G = 8;
    // small batches: fewer samples per CTA so that the grid still covers the SMs; the N = 32 launch of a
    // cfg-3 rank is 16 CTAs of 2 samples instead of 4 CTAs of 8, and its phase Q is 4x shorter
    const int64_t want_ctas = (int64_t)sm_count();
    while (G > 2 && ceil_div(q.N, G) < want_ctas) G -= 2;
    while (G > 1 && need(G) > (size_t)75 * 1024) --G;
    const size_t smem = need(G);
    if (smem > (size_t)smem_limit()) return MR_ERR_UNSUPPORTED;
    q.G = G;
    q.vec = pick_vec<float>(lp, q.N, q.C, G);
    if (MODE == MODE_GRAD && ((uintptr_t)grad % 16) != 0) q.vec = 1;
    const int pitch = pitch_of(G);
    if (pitch % 4) q.vec = 1;
    if (MODE != MODE_GRAD && ((uintptr_t)fac % 16) != 0) q.vec = 1;
    auto kern = (q.H == 8) ? ctc2d_dp4_kernel<MODE, 8> : ctc2d_dp4_kernel<MODE, 0>;
    { int rc_attr = ensure_dyn_smem((const void *)kern, smem, "ctc2d_dp4 attr"); if (rc_attr) return rc_attr; }
    kern<<<(unsigned)ceil_div(q.N, q.G), 256, smem, st>>>(q, lp, tg, il, tl, go, go_stride, nll, fac, grad, pitch);
    return check_launch("ctc2d_dp4_kernel");
}

template <int MODE>
int launch_dpg(Geo q, const float *lp, const int64_t *tg, const int64_t *il, const int64_t *tl, const float *go,
               int64_t go_stride, float *nll, float *fac, float *grad, cudaStream_t st) {
    if (MODE == MODE_FAC_STD || q.S > 32) return MR_ERR_UNSUPPORTED;
    const size_t smem = 4 * sizeof(float) * ((size_t)q.T * (33 + 99) + 96);
    if (smem > (size_t)smem_limit()) return MR_ERR_UNSUPPORTED;
    auto kern = ctc2d_dpg_kernel<MODE>;
    { int rc_attr = ensure_dyn_smem((const void *)kern, smem, "ctc2d_dpg attr"); if (rc_attr) return rc_attr; }
    kern<<<(unsigned)ceil_div(q.N, 4), 128, smem, st>>>(q, lp, tg, il, tl, go, go_stride, nll, fac, grad);
    return check_launch("ctc2d_dpg_kernel");
}

template <typename real, bool FAST, int MODE>
int launch_dp(const real *lp, const int64_t *tg, const int64_t *il, const int64_t *tl, const real *go,
              int64_t go_stride, int64_t T, int64_t H, int64_t N, int64_t C, int64_t S, int64_t tg_sn,
              int64_t tg_ss, int64_t blank, real *nll, real *fac, real *grad, cudaStream_t st, int zero_inf = 0) {
    Geo q;
    q.zero_inf = zero_inf;
    q.T = (int)T; q.H = (int)H; q.N = (int)N; q.C = (int)C; q.S = (int)S; q.SS = (int)(2 * S + 1);
    q.blank = (int)blank; q.tg_sn = tg_sn; q.tg_ss = tg_ss;
    // fp32 fast-math requests use the warp-per-sample kernel (MR_CTC2D_BLOCK_DP=1 forces the block variant below);
    // accurate-math and fp64 requests, and shapes whose plan does not fit, use the block variant.
    if (sizeof(real) == 4 && FAST && MODE != MODE_FAC_STD && !getenv("MR_CTC2D_BLOCK_DP") && !getenv("MR_CTC2D_DP_V3")) {
        q.G = 8; q.vec = 1;
        int rc = launch_dp4<MODE>(q, (const float *)lp, tg, il, tl, (const float *)go, go_stride, (float *)nll,
                                  (float *)fac, (float *)grad, st);
        if (rc != MR_ERR_UNSUPPORTED) return rc;
        if (q.C > 64) {   // large alphabet: gather kernel (nothing of size C on chip)
            rc = launch_dpg<MODE>(q, (const float *)lp, tg, il, tl, (const float *)go, go_stride, (float *)nll,
                                  (float *)fac, (float *)grad, st);
            if (rc != MR_ERR_UNSUPPORTED) return rc;
        }
    }
    if (sizeof(real) == 4 && FAST && !getenv("MR_CTC2D_BLOCK_DP")) {
        q.G = 8; q.vec = 1;
        const int rc = launch_dp_warp<MODE>(q, (const float *)lp, tg, il, tl, (const float *)go, go_stride, (float *)nll,
                                            (float *)fac, (float *)grad, st);
        if (rc != MR_ERR_UNSUPPORTED) return rc;
    }
    int G = 160 / q.SS;  // fewer samples per CTA than the alpha kernel: the sweeps are latency-bound,
    if (G < 1) G = 1;    // more co-resident CTAs keep HBM busy meanwhile
    if (G > 8) G = 8;
    auto need = [&](int g) {
        return sizeof(real) * ((size_t)2 * T * g * C + (size_t)T * g * q.SS + (size_t)2 * g * q.SS + 3 * g) +
               (size_t)T * g * C + 16;
    };
    while (G > 1 && need(G) > (size_t)44 * 1024) --G;
    const size_t smem = need(G);
    if (smem > (size_t)smem_limit()) return MR_ERR_UNSUPPORTED;
    q.G = G;
    q.vec = pick_vec<real>(lp, N, C, G);
    if (MODE == MODE_GRAD && ((uintptr_t)grad % 16) != 0) q.vec = 1;
    const int threads = (int)round_up((int64_t)G * q.SS, 32);
    const int grid = (int)ceil_div(N, G);
    auto kern = (H == 8) ? ctc2d_dp_kernel<real, FAST, MODE, 8> : ctc2d_dp_kernel<real, FAST, MODE, 0>;
    if (smem > 48 * 1024)
        MR_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "ctc2d_dp attr");
    kern<<<grid, threads, smem, st>>>(q, lp, tg, il, tl, go, go_stride, nll, fac, grad);
    return check_launch("ctc2d_dp_kernel");
}

}  // namespace

extern "C" {

int mr_ctc2d_forward_f32(const float *lp, const int64_t *tg, const int64_t *il, const int64_t *tl, int64_t T,
                         int64_t H, int64_t N, int64_t C, int64_t S, int64_t tg_sn, int64_t tg_ss, int64_t blank,
                         int fast_math, float *nll, float *la, void *stream) {
    int rc = check_common(lp, tg, il, tl, T, H, N, C, S, blank);
    if (rc) return rc;
    if (N == 0) return MR_OK;
    if (T == 0 || H == 0) return MR_ERR_BAD_SHAPE;
    if (!nll || !la) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    return fast_math ? launch_alpha<float, true>(lp, tg, il, tl, T, H, N, C, S, tg_sn, tg_ss, blank, nll, la, st)
                     : launch_alpha<float, false>(lp, tg, il, tl, T, H, N, C, S, tg_sn, tg_ss, blank, nll, la, st);
}

int mr_ctc2d_forward_f64(const double *lp, const int64_t *tg, const int64_t *il, const int64_t *tl, int64_t T,
                         int64_t H, int64_t N, int64_t C, int64_t S, int64_t tg_sn, int64_t tg_ss, int64_t blank,
                         int fast_math, double *nll, double *la, void *stream) {
    (void)fast_math;
    int rc = check_common(lp, tg, il, tl, T, H, N, C, S, blank);
    if (rc) return rc;
    if (N == 0) return MR_OK;
    if (T == 0 || H == 0) return MR_ERR_BAD_SHAPE;
    if (!nll || !la) return MR_ERR_NULL_POINTER;
    return launch_alpha<double, false>(lp, tg, il, tl, T, H, N, C, S, tg_sn, tg_ss, blank, nll, la, (cudaStream_t)stream);
}

int mr_ctc2d_backward_f32(const float *go, int64_t go_stride, const float *lp, const int64_t *tg, const int64_t *il,
                          const int64_t *tl, const float *nll, const float *la, int64_t T, int64_t H, int64_t N,
                          int64_t C, int64_t S, int64_t tg_sn, int64_t tg_ss, int64_t blank, int fast_math,
                          float *grad, void *stream) {
    (void)nll; (void)la;
    int rc = check_common(lp, tg, il, tl, T, H, N, C, S, blank);
    if (rc) return rc;
    if (N == 0 || T == 0 || H == 0) return MR_OK;
    if (!go || !grad) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    return fast_math ? launch_dp<float, true, MODE_GRAD>(lp, tg, il, tl, go, go_stride, T, H, N, C, S, tg_sn, tg_ss, blank, nullptr, nullptr, grad, st)
                     : launch_dp<float, false, MODE_GRAD>(lp, tg, il, tl, go, go_stride, T, H, N, C, S, tg_sn, tg_ss, blank, nullptr, nullptr, grad, st);
}

int mr_ctc2d_backward_f64(const double *go, int64_t go_stride, const double *lp, const int64_t *tg, const int64_t *il,
                          const int64_t *tl, const double *nll, const double *la, int64_t T, int64_t H, int64_t N,
                          int64_t C, int64_t S, int64_t tg_sn, int64_t tg_ss, int64_t blank, int fast_math,
                          double *grad, void *stream) {
    (void)nll; (void)la; (void)fast_math;
    int rc = check_common(lp, tg, il, tl, T, H, N, C, S, blank);
    if (rc) return rc;
    if (N == 0 || T == 0 || H == 0) return MR_OK;
    if (!go || !grad) return MR_ERR_NULL_POINTER;
    return launch_dp<double, false, MODE_GRAD>(lp, tg, il, tl, go, go_stride, T, H, N, C, S, tg_sn, tg_ss, blank, nullptr, nullptr, grad, (cudaStream_t)stream);
}

int mr_ctc2d_forward_train_f32(const float *lp, const int64_t *tg, const int64_t *il, const int64_t *tl, int64_t T,
                               int64_t H, int64_t N, int64_t C, int64_t S, int64_t tg_sn, int64_t tg_ss,
                               int64_t blank, int fast_math, float *nll, float *gfac, void *stream) {
    int rc = check_common(lp, tg, il, tl, T, H, N, C, S, blank);
    if (rc) return rc;
    if (N == 0) return MR_OK;
    if (T == 0 || H == 0) return MR_ERR_BAD_SHAPE;
    if (!nll || !gfac) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    return fast_math ? launch_dp<float, true, MODE_FAC>(lp, tg, il, tl, nullptr, 0, T, H, N, C, S, tg_sn, tg_ss, blank, nll, gfac, nullptr, st)
                     : launch_dp<float, false, MODE_FAC>(lp, tg, il, tl, nullptr, 0, T, H, N, C, S, tg_sn, tg_ss, blank, nll, gfac, nullptr, st);
}

int mr_ctc2d_backward_apply_f32(const float *go, int64_t go_stride, const float *lp, const float *gfac, int64_t T,
                                int64_t H, int64_t N, int64_t C, int fast_math, float *grad, void *stream) {
    if (T < 0 || H < 0 || N < 0 || C <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0 || T == 0 || H == 0) return MR_OK;
    if (!go || !lp || !gfac || !grad) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    const bool v4 = ((uintptr_t)lp % 16 == 0) && ((uintptr_t)grad % 16 == 0) && ((uintptr_t)gfac % 16 == 0) && ((N * C) % 4 == 0);
    const int64_t nvec_row = N * C / (v4 ? 4 : 1);
    const int threads = 256;
    int64_t bx = ceil_div(nvec_row, threads);
    if (bx > 65535) bx = 65535;
    if (T > 65535) return MR_ERR_BAD_SHAPE;
    dim3 grid((unsigned)bx, (unsigned)T);
#define MR_APPLY(FASTV, VEV, HTV) ctc2d_apply_kernel<FASTV, VEV, HTV><<<grid, threads, 0, st>>>(lp, gfac, go, go_stride, (int)T, (int)H, (int)N, (int)C, grad)
    if (v4) {
        if (H == 8) { if (fast_math) MR_APPLY(true, 4, 8); else MR_APPLY(false, 4, 8); }
        else { if (fast_math) MR_APPLY(true, 4, 0); else MR_APPLY(false, 4, 0); }
    } else {
        if (fast_math) MR_APPLY(true, 1, 0); else MR_APPLY(false, 1, 0);
    }
#undef MR_APPLY
    return check_launch("ctc2d_apply_kernel");
}


/* ---------------- 1D CTC (CRNN head): log_softmax rows -> DP (H = 1) -> gradient w.r.t. the logits ------------- */

int mr_log_softmax_rows_f32(const float *x, int64_t rows, int64_t C, float *out, void *stream) {
    if (rows < 0 || C <= 0) return MR_ERR_BAD_SHAPE;
    if (rows == 0) return MR_OK;
    if (!x || !out) return MR_ERR_NULL_POINTER;
    const int wpb = 8;
    rows_log_softmax_kernel<<<(unsigned)ceil_div(rows, wpb), wpb * 32, 0, (cudaStream_t)stream>>>(x, rows, (int)C, out);
    return check_launch("rows_log_softmax_kernel");
}

int mr_ctc1d_forward_train_f32(const float *log_probs, const int64_t *tg, const int64_t *il, const int64_t *tl,
                               int64_t T, int64_t N, int64_t C, int64_t S, int64_t tg_sn, int64_t tg_ss, int64_t blank,
                               int zero_infinity, int fast_math, float *nll, float *gfac, void *stream) {
    int rc = check_common(log_probs, tg, il, tl, T, 1, N, C, S, blank);
    if (rc) return rc;
    if (N == 0) return MR_OK;
    if (T == 0) return MR_ERR_BAD_SHAPE;
    if (!nll || !gfac) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    return fast_math ? launch_dp<float, true, MODE_FAC_STD>(log_probs, tg, il, tl, nullptr, 0, T, 1, N, C, S, tg_sn, tg_ss, blank, nll, gfac, nullptr, st, zero_infinity)
                     : launch_dp<float, false, MODE_FAC_STD>(log_probs, tg, il, tl, nullptr, 0, T, 1, N, C, S, tg_sn, tg_ss, blank, nll, gfac, nullptr, st, zero_infinity);
}

int mr_ctc1d_backward_logits_f32(const float *log_probs, const float *gfac, const float *scale, int64_t T, int64_t N,
                                 int64_t C, float *grad_logits, void *stream) {
    if (T < 0 || N < 0 || C <= 0) return MR_ERR_BAD_SHAPE;
    if (T == 0 || N == 0) return MR_OK;
    if (!log_probs || !gfac || !scale || !grad_logits) return MR_ERR_NULL_POINTER;
    const int wpb = 8;
    ctc1d_grad_rows_kernel<<<(unsigned)ceil_div(T * N, wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
        log_probs, gfac, scale, T * N, (int)N, (int)C, grad_logits);
    return check_launch("ctc1d_grad_rows_kernel");
}

}  // extern "C"
