// Deformable convolution v1 / v2 (modulated) for sm_90a, fp32, NCHW — replaces the reference extension
// `deform_conv_cuda` (assets/ops/dcn/src/deform_conv_cuda.cpp:151-695, deform_conv_cuda_kernel.cu K5-K10).
//
// Not a port.  The reference loops over the batch on the host (1 im2col launch + G GEMMs per sample,
// deform_conv_cuda.cpp:534-550) and runs one thread per (channel, pixel) that re-derives the nine sampling
// positions for every channel.  Here:
//   * dcn_im2col_kernel     one thread = one sampling point (sample, deformable group, tap k, pixel p); the four
//                           bilinear corner offsets / weights are computed ONCE and reused for every channel of the
//                           group, so the inner loop is 4 cached gathers + 1 coalesced store per channel.  All
//                           samples of a chunk go in one launch; the GEMM is one strided-batched cuBLAS SGEMM.
//   * dcn_col2im_kernel     the reference's K9 (grad_input scatter) and K10 (grad_offset + grad_mask) fused:
//                           the W^T.grad_out columns are read once, both offset components and the mask gradient
//                           come out of the same loop.
//   * dcn_bias_grad_kernel  per-channel sum of grad_output (the reference's GEMM with a ones vector, :659-665).
// Indexing quirks kept on purpose (SURVEY.md App. B2): offset / mask (and their gradients) are addressed per
// sample as base + b*batch_stride and then FLAT with (Ho, Wo) strides (deform_conv_cuda_kernel.cu:599-609,
// :761-764), whatever spatial size the caller's tensors have.
//
// Roofline: the gather/scatter kernels are HBM-bound on the column matrix (9*C*Ho*Wo*4 B per sample written,
// then read by the GEMM); the GEMMs are plain fp32 library GEMMs (cuBLAS, no TF32: parity is 1e-4).
#include "common.cuh"
#include <math.h>

namespace {
using namespace mr;

struct DcnGeo {
    int B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg, Ho, Wo;
    int K, P, cpg;  // taps, output pixels, channels per deformable group
    int64_t off_bs, mask_bs, goff_bs, gmask_bs;
};

struct Tap {
    int o1, o2, o3, o4;       // corner offsets inside one channel plane (0 when the corner is outside)
    float w1, w2, w3, w4;     // bilinear weights, zeroed for corners outside the image
    float lh, lw;             // fractional parts (for the coordinate gradient)
    bool m1, m2, m3, m4;      // corner inside the image
    bool inside;              // sampling point in (-1, H) x (-1, W)   (deform_conv_cuda_kernel.cu:617)
};

// dmcn_im2col_bilinear (deform_conv_cuda_kernel.cu:466-496) split into setup + per-channel evaluation
__device__ __forceinline__ Tap make_tap(float h, float w, int H, int W) {
    Tap t;
    t.inside = (h > -1.f && w > -1.f && h < (float)H && w < (float)W);
    const int hl = (int)floorf(h), wl = (int)floorf(w);
    const int hh = hl + 1, wh = wl + 1;
    t.lh = h - hl;
    t.lw = w - wl;
    const float uh = 1.f - t.lh, uw = 1.f - t.lw;
    t.m1 = t.inside && hl >= 0 && wl >= 0;
    t.m2 = t.inside && hl >= 0 && wh <= W - 1;
    t.m3 = t.inside && hh <= H - 1 && wl >= 0;
    t.m4 = t.inside && hh <= H - 1 && wh <= W - 1;
    t.o1 = t.m1 ? hl * W + wl : 0;
    t.o2 = t.m2 ? hl * W + wh : 0;
    t.o3 = t.m3 ? hh * W + wl : 0;
    t.o4 = t.m4 ? hh * W + wh : 0;
    t.w1 = t.m1 ? uh * uw : 0.f;
    t.w2 = t.m2 ? uh * t.lw : 0.f;
    t.w3 = t.m3 ? t.lh * uw : 0.f;
    t.w4 = t.m4 ? t.lh * t.lw : 0.f;
    return t;
}

// One thread per (sample in chunk, channel slice, deformable group, tap, pixel).
__global__ void __launch_bounds__(256)
dcn_im2col_kernel(DcnGeo g, int b0, int nb, int csplit, const float *__restrict__ input,
                  const float *__restrict__ offset, const float *__restrict__ mask, float *__restrict__ col) {
    const int64_t total = (int64_t)nb * csplit * g.dg * g.K * g.P;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int p = (int)(idx % g.P);
        int64_t r = idx / g.P;
        const int k = (int)(r % g.K); r /= g.K;
        const int dgi = (int)(r % g.dg); r /= g.dg;
        const int cs = (int)(r % csplit);
        const int bl = (int)(r / csplit);
        const int b = b0 + bl;
        const int ho = p / g.Wo, wo = p - ho * g.Wo;
        const int i = k / g.kw, j = k - i * g.kw;
        const float *offp = offset + (int64_t)b * g.off_bs + (int64_t)dgi * 2 * g.K * g.P;
        const float oh = __ldg(offp + (int64_t)(2 * k) * g.P + p);
        const float ow = __ldg(offp + (int64_t)(2 * k + 1) * g.P + p);
        const float m = mask ? __ldg(mask + (int64_t)b * g.mask_bs + (int64_t)(dgi * g.K + k) * g.P + p) : 1.f;
        const float h_im = (float)(ho * g.sh - g.ph + i * g.dh) + oh;
        const float w_im = (float)(wo * g.sw - g.pw + j * g.dw) + ow;
        const Tap t = make_tap(h_im, w_im, g.H, g.W);
        const int per = (g.cpg + csplit - 1) / csplit;
        const int c_lo = dgi * g.cpg + cs * per;
        const int c_hi = min(dgi * g.cpg + g.cpg, c_lo + per);
        const int64_t plane = (int64_t)g.H * g.W;
        const float *im = input + ((int64_t)b * g.C + c_lo) * plane;
        float *out = col + (((int64_t)bl * g.C + c_lo) * g.K + k) * g.P + p;
        const int64_t ostep = (int64_t)g.K * g.P;
#pragma unroll 4
        for (int c = c_lo; c < c_hi; ++c) {
            const float v = t.w1 * __ldg(im + t.o1) + t.w2 * __ldg(im + t.o2) + t.w3 * __ldg(im + t.o3) +
                            t.w4 * __ldg(im + t.o4);
            __stcs(out, v * m);
            im += plane;
            out += ostep;
        }
    }
}

// K9 + K10 fused.  colg = W^T . grad_output for the chunk, [nb][C*K][P].
__global__ void __launch_bounds__(256)
dcn_col2im_kernel(DcnGeo g, int b0, int nb, const float *__restrict__ colg, const float *__restrict__ input,
                  const float *__restrict__ offset, const float *__restrict__ mask, float *__restrict__ grad_input,
                  float *__restrict__ grad_offset, float *__restrict__ grad_mask) {
    const int64_t total = (int64_t)nb * g.dg * g.K * g.P;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int p = (int)(idx % g.P);
        int64_t r = idx / g.P;
        const int k = (int)(r % g.K); r /= g.K;
        const int dgi = (int)(r % g.dg);
        const int bl = (int)(r / g.dg);
        const int b = b0 + bl;
        const int ho = p / g.Wo, wo = p - ho * g.Wo;
        const int i = k / g.kw, j = k - i * g.kw;
        const float *offp = offset + (int64_t)b * g.off_bs + (int64_t)dgi * 2 * g.K * g.P;
        const float oh = __ldg(offp + (int64_t)(2 * k) * g.P + p);
        const float ow = __ldg(offp + (int64_t)(2 * k + 1) * g.P + p);
        const float m = mask ? __ldg(mask + (int64_t)b * g.mask_bs + (int64_t)(dgi * g.K + k) * g.P + p) : 1.f;
        const float h_im = (float)(ho * g.sh - g.ph + i * g.dh) + oh;
        const float w_im = (float)(wo * g.sw - g.pw + j * g.dw) + ow;
        const Tap t = make_tap(h_im, w_im, g.H, g.W);
        const float uh = 1.f - t.lh, uw = 1.f - t.lw;
        const int c_lo = dgi * g.cpg;
        const int64_t plane = (int64_t)g.H * g.W;
        const float *im = input + ((int64_t)b * g.C + c_lo) * plane;
        float *gim = grad_input ? grad_input + ((int64_t)b * g.C + c_lo) * plane : nullptr;
        const float *cg = colg + (((int64_t)bl * g.C + c_lo) * g.K + k) * g.P + p;
        const int64_t cstep = (int64_t)g.K * g.P;
        float val_h = 0.f, val_w = 0.f, mval = 0.f;
        if (t.inside) {
            for (int c = 0; c < g.cpg; ++c) {
                const float gcol = __ldcs(cg);
                const float v1 = t.m1 ? __ldg(im + t.o1) : 0.f;
                const float v2 = t.m2 ? __ldg(im + t.o2) : 0.f;
                const float v3 = t.m3 ? __ldg(im + t.o3) : 0.f;
                const float v4 = t.m4 ? __ldg(im + t.o4) : 0.f;
                // K10 :752 (mask gradient) and dmcn_get_coordinate_weight :527-567
                mval += gcol * (t.w1 * v1 + t.w2 * v2 + t.w3 * v3 + t.w4 * v4);
                const float gm = gcol * m;
                val_h += (uw * (v3 - v1) + t.lw * (v4 - v2)) * gm;
                val_w += (uh * (v2 - v1) + t.lh * (v4 - v3)) * gm;
                // K9 :676-690: bilinear scatter of col*mask onto the (valid) corners
                if (gim) {
                    if (t.m1) atomicAdd(gim + t.o1, t.w1 * gm);
                    if (t.m2) atomicAdd(gim + t.o2, t.w2 * gm);
                    if (t.m3) atomicAdd(gim + t.o3, t.w3 * gm);
                    if (t.m4) atomicAdd(gim + t.o4, t.w4 * gm);
                    gim += plane;
                }
                im += plane;
                cg += cstep;
            }
        }
        if (grad_offset) {
            float *go = grad_offset + (int64_t)b * g.goff_bs + (int64_t)dgi * 2 * g.K * g.P;
            go[(int64_t)(2 * k) * g.P + p] = val_h;
            go[(int64_t)(2 * k + 1) * g.P + p] = val_w;
        }
        if (grad_mask) grad_mask[(int64_t)b * g.gmask_bs + (int64_t)(dgi * g.K + k) * g.P + p] = mval;
    }
}

// grad_bias[o] += sum_{b,p} grad_output[b,o,p]  (one CTA per output channel)
__global__ void dcn_bias_grad_kernel(const float *__restrict__ go, int B, int Cout, int P, float *__restrict__ gb) {
    const int o = blockIdx.x;
    float acc = 0.f;
    for (int64_t i = threadIdx.x; i < (int64_t)B * P; i += blockDim.x) {
        const int b = (int)(i / P);
        const int p = (int)(i - (int64_t)b * P);
        acc += go[((int64_t)b * Cout + o) * P + p];
    }
    __shared__ float red[32];
    for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        acc = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
        if (threadIdx.x == 0) gb[o] += acc;
    }
}

__global__ void dcn_bias_add_kernel(float *__restrict__ out, const float *__restrict__ bias, int Cout, int P, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] += bias[(i / P) % Cout];
}

int fill_geo(DcnGeo &g, int B, int C, int H, int W, int Cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh,
             int dw, int group, int dg) {
    if (B < 0 || C <= 0 || H <= 0 || W <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || dh <= 0 ||
        dw <= 0 || ph < 0 || pw < 0 || group <= 0 || dg <= 0)
        return MR_ERR_BAD_SHAPE;
    if (C % group || Cout % group || C % dg) return MR_ERR_BAD_SHAPE;
    g.B = B; g.C = C; g.H = H; g.W = W; g.Cout = Cout; g.kh = kh; g.kw = kw; g.sh = sh; g.sw = sw; g.ph = ph;
    g.pw = pw; g.dh = dh; g.dw = dw; g.group = group; g.dg = dg;
    g.Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;
    g.Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
    if (g.Ho <= 0 || g.Wo <= 0) return MR_ERR_BAD_SHAPE;
    g.K = kh * kw; g.P = g.Ho * g.Wo; g.cpg = C / dg;
    g.off_bs = g.mask_bs = g.goff_bs = g.gmask_bs = 0;
    return MR_OK;
}

int grid_for(int64_t threads_total, int block) {
    int64_t blocks = ceil_div(threads_total, block);
    const int64_t cap = (int64_t)mr::sm_count() * 32;
    return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

int pick_csplit(const DcnGeo &g, int nb) {
    // enough sampling points to fill the chip? otherwise slice the channel loop
    const int64_t pts = (int64_t)nb * g.dg * g.K * g.P;
    int cs = 1;
    while (pts * cs < mr::sm_count() * 2048 * 2 && cs * 2 <= g.cpg && cs < 32) cs *= 2;
    return cs;
}

}  // namespace

extern "C" {

int64_t mr_dcn_workspace_bytes(int64_t nb, int64_t C, int64_t kh, int64_t kw, int64_t Ho, int64_t Wo) {
    return nb * C * kh * kw * Ho * Wo * (int64_t)sizeof(float);
}

int mr_dcn_forward_f32(const float *input, const float *weight, const float *bias, const float *offset,
                       int64_t offset_bstride, const float *mask, int64_t mask_bstride, float *output,
                       float *workspace, int64_t workspace_bytes, int B, int C, int H, int W, int Cout, int kh, int kw,
                       int sh, int sw, int ph, int pw, int dh, int dw, int group, int dg, void *stream) {
    DcnGeo g;
    int rc = fill_geo(g, B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg);
    if (rc) return rc;
    if (B == 0) return MR_OK;
    if (!input || !weight || !offset || !output || !workspace) return MR_ERR_NULL_POINTER;
    // fused wgmma implicit GEMM (csrc/dcn_tcgen05.cu) when the shape qualifies and the workspace holds its scratch
    rc = mr_dcn_forward_fused_f32(input, weight, bias, offset, offset_bstride, mask, mask_bstride, output, workspace,
                                  workspace_bytes, B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg, stream);
    if (rc != MR_ERR_UNSUPPORTED) return rc;
    g.off_bs = offset_bstride; g.mask_bs = mask_bstride;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t per = mr_dcn_workspace_bytes(1, C, kh, kw, g.Ho, g.Wo);
    const int chunk = (int)(workspace_bytes / per < B ? workspace_bytes / per : B);
    if (chunk < 1) return MR_ERR_BAD_SHAPE;
    cublasHandle_t h;
    rc = blas_handle(&h, st);
    if (rc) return rc;
    const int Cg = C / group, Og = Cout / group, CgK = Cg * g.K;
    const float one = 1.f, zero = 0.f;
    for (int b0 = 0; b0 < B; b0 += chunk) {
        const int nb = (B - b0 < chunk) ? B - b0 : chunk;
        const int cs = pick_csplit(g, nb);
        dcn_im2col_kernel<<<grid_for((int64_t)nb * cs * g.dg * g.K * g.P, 256), 256, 0, st>>>(g, b0, nb, cs, input, offset, mask, workspace);
        rc = check_launch("dcn_im2col_kernel");
        if (rc) return rc;
        for (int gr = 0; gr < group; ++gr) {
            // out[b][gr] (Og x P) = W[gr] (Og x CgK) . col[b][gr] (CgK x P)   (row-major) -- deform_conv_cuda.cpp:545-550
            MR_BLAS_TRY(cublasSgemmStridedBatched(h, CUBLAS_OP_N, CUBLAS_OP_N, g.P, Og, CgK, &one,
                                                  workspace + (int64_t)gr * CgK * g.P, g.P, (int64_t)C * g.K * g.P,
                                                  weight + (int64_t)gr * Og * CgK, CgK, 0, &zero,
                                                  output + ((int64_t)b0 * Cout + gr * Og) * g.P, g.P, (int64_t)Cout * g.P, nb),
                        "cublasSgemmStridedBatched(dcn forward)");
        }
    }
    if (bias) {
        const int64_t n = (int64_t)B * Cout * g.P;
        dcn_bias_add_kernel<<<grid_for(n, 256), 256, 0, st>>>(output, bias, Cout, g.P, n);
        rc = check_launch("dcn_bias_add_kernel");
        if (rc) return rc;
    }
    return MR_OK;
}

int mr_dcn_backward_f32(const float *input, const float *weight, const float *offset, int64_t offset_bstride,
                        const float *mask, int64_t mask_bstride, const float *grad_output, float *grad_input,
                        float *grad_weight, float *grad_bias, float *grad_offset, int64_t grad_offset_bstride,
                        float *grad_mask, int64_t grad_mask_bstride, float weight_grad_scale, float *workspace,
                        int64_t workspace_bytes, int B, int C, int H, int W, int Cout, int kh, int kw, int sh, int sw,
                        int ph, int pw, int dh, int dw, int group, int dg, void *stream) {
    DcnGeo g;
    int rc = fill_geo(g, B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg);
    if (rc) return rc;
    if (B == 0) return MR_OK;
    if (!input || !weight || !offset || !grad_output || !workspace) return MR_ERR_NULL_POINTER;
    g.off_bs = offset_bstride; g.mask_bs = mask_bstride; g.goff_bs = grad_offset_bstride; g.gmask_bs = grad_mask_bstride;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t per = mr_dcn_workspace_bytes(1, C, kh, kw, g.Ho, g.Wo);
    const int chunk = (int)(workspace_bytes / per < B ? workspace_bytes / per : B);
    if (chunk < 1) return MR_ERR_BAD_SHAPE;
    cublasHandle_t h;
    rc = blas_handle(&h, st);
    if (rc) return rc;
    const int Cg = C / group, Og = Cout / group, CgK = Cg * g.K;
    const float one = 1.f, zero = 0.f;
    const bool want_data = grad_input || grad_offset || grad_mask;
    bool wgrad_done = false;
    // everything but grad_bias on the fused wgmma kernels when the shape allows (csrc/dcn_tcgen05.cu)
    rc = mr_dcn_backward_fused_f32(input, weight, offset, offset_bstride, mask, mask_bstride, grad_output, grad_input, grad_weight,
                                   grad_offset, grad_offset_bstride, grad_mask, grad_mask_bstride, weight_grad_scale, workspace,
                                   workspace_bytes, B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg, stream);
    if (rc != MR_OK && rc != MR_ERR_UNSUPPORTED) return rc;
    const bool fused_all = rc == MR_OK;
    if (grad_weight && !fused_all) {
        // fused wgmma weight gradient (csrc/dcn_tcgen05.cu): uses the workspace first; the loop below reuses it afterwards
        rc = mr_dcn_wgrad_fused_f32(input, offset, offset_bstride, mask, mask_bstride, grad_output, grad_weight, weight_grad_scale,
                                    workspace, workspace_bytes, B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg, stream);
        if (rc == MR_OK) wgrad_done = true;
        else if (rc != MR_ERR_UNSUPPORTED) return rc;
    }
    for (int b0 = 0; b0 < B && !fused_all; b0 += chunk) {
        const int nb = (B - b0 < chunk) ? B - b0 : chunk;
        if (want_data) {
            for (int gr = 0; gr < group; ++gr) {
                // colg[b][gr] (CgK x P) = W[gr]^T (CgK x Og) . go[b][gr] (Og x P)          -- :611-614
                MR_BLAS_TRY(cublasSgemmStridedBatched(h, CUBLAS_OP_N, CUBLAS_OP_T, g.P, CgK, Og, &one,
                                                      grad_output + ((int64_t)b0 * Cout + gr * Og) * g.P, g.P, (int64_t)Cout * g.P,
                                                      weight + (int64_t)gr * Og * CgK, CgK, 0, &zero,
                                                      workspace + (int64_t)gr * CgK * g.P, g.P, (int64_t)C * g.K * g.P, nb),
                            "cublasSgemmStridedBatched(dcn colgrad)");
            }
            dcn_col2im_kernel<<<grid_for((int64_t)nb * g.dg * g.K * g.P, 256), 256, 0, st>>>(
                g, b0, nb, workspace, input, offset, mask, grad_input, grad_offset, grad_mask);
            rc = check_launch("dcn_col2im_kernel");
            if (rc) return rc;
        }
        if (grad_weight && !wgrad_done) {
            const int cs = pick_csplit(g, nb);
            dcn_im2col_kernel<<<grid_for((int64_t)nb * cs * g.dg * g.K * g.P, 256), 256, 0, st>>>(g, b0, nb, cs, input, offset, mask, workspace);
            rc = check_launch("dcn_im2col_kernel");
            if (rc) return rc;
            for (int bl = 0; bl < nb; ++bl)
                for (int gr = 0; gr < group; ++gr) {
                    // gw[gr] (Og x CgK) += scale * go[b][gr] (Og x P) . col[b][gr]^T (P x CgK)   -- :653-658
                    MR_BLAS_TRY(cublasSgemm(h, CUBLAS_OP_T, CUBLAS_OP_N, CgK, Og, g.P, &weight_grad_scale,
                                            workspace + ((int64_t)bl * C * g.K + (int64_t)gr * CgK) * g.P, g.P,
                                            grad_output + ((int64_t)(b0 + bl) * Cout + gr * Og) * g.P, g.P, &one,
                                            grad_weight + (int64_t)gr * Og * CgK, CgK),
                                "cublasSgemm(dcn wgrad)");
                }
        }
    }
    if (grad_bias) {
        dcn_bias_grad_kernel<<<Cout, 256, 0, st>>>(grad_output, B, Cout, g.P, grad_bias);
        rc = check_launch("dcn_bias_grad_kernel");
        if (rc) return rc;
    }
    return MR_OK;
}

}  // extern "C"
