// Deformable position-sensitive RoI pooling for sm_90a (SURVEY.md section 8 rows A13 / N4): replaces
// assets/ops/dcn/src/deform_pool_cuda_kernel.cu:52-263 + deform_pool_cuda.cpp:29-81 behind the same five-plus-arguments
// surface (functions/deform_pool.py:7-69).  fp32.
//
// The op is a sparse gather: every output bin (roi n, channel c, bin ph, pw) averages sample_per_part^2 bilinear
// samples of ONE position-sensitive input plane, optionally shifted by a learned per-part offset.  Nothing is reused
// between bins except the RoI record, so the mapping is one thread per output bin (consecutive threads = consecutive
// pw, i.e. neighbouring sample positions in the same plane: the gathers of a warp land in a few cache lines).  The
// backward scatters with fp32 atomics (different RoIs overlap arbitrarily) and adds the offset gradient from the same
// four corner values.  Forward and backward share one geometry routine so they cannot drift apart.
#include "common.cuh"
#include <math.h>

namespace {
using namespace mr;

struct PoolArgs {
    int channels, height, width, num_rois, no_trans, output_dim, group_size, pooled, part_size, sample_per_part;
    int num_classes, channels_each_class;
    float spatial_scale, trans_std;
};

struct Bin {
    int batch, chan, tx_index, ty_index;
    float roi_w, roi_h, wstart, hstart, sub_w, sub_h;
};

// geometry of output element `index` = ((n * output_dim + ctop) * P + ph) * P + pw      (kernel.cu:71-116)
__device__ __forceinline__ Bin bin_geometry(const PoolArgs &a, const float *__restrict__ rois, const float *__restrict__ trans,
                                            int64_t index) {
    const int P = a.pooled;
    const int pw = (int)(index % P), ph = (int)((index / P) % P);
    const int ctop = (int)((index / P / P) % a.output_dim), n = (int)(index / P / P / a.output_dim);
    Bin b;
    const float *r = rois + (int64_t)n * 5;
    b.batch = (int)r[0];
    const float start_w = roundf(r[1]) * a.spatial_scale - 0.5f, start_h = roundf(r[2]) * a.spatial_scale - 0.5f;
    const float end_w = (roundf(r[3]) + 1.f) * a.spatial_scale - 0.5f, end_h = (roundf(r[4]) + 1.f) * a.spatial_scale - 0.5f;
    b.roi_w = fmaxf(end_w - start_w, 0.1f);
    b.roi_h = fmaxf(end_h - start_h, 0.1f);
    const float bin_h = b.roi_h / (float)P, bin_w = b.roi_w / (float)P;
    b.sub_h = bin_h / (float)a.sample_per_part;
    b.sub_w = bin_w / (float)a.sample_per_part;
    const int part_h = (int)floorf((float)ph / P * a.part_size), part_w = (int)floorf((float)pw / P * a.part_size);
    const int class_id = ctop / a.channels_each_class;
    float tx = 0.f, ty = 0.f;
    b.tx_index = b.ty_index = -1;
    if (!a.no_trans) {
        b.tx_index = (((n * a.num_classes + class_id) * 2) * a.part_size + part_h) * a.part_size + part_w;
        b.ty_index = (((n * a.num_classes + class_id) * 2 + 1) * a.part_size + part_h) * a.part_size + part_w;
        tx = trans[b.tx_index] * a.trans_std;
        ty = trans[b.ty_index] * a.trans_std;
    }
    b.wstart = (float)pw * bin_w + start_w + tx * b.roi_w;
    b.hstart = (float)ph * bin_h + start_h + ty * b.roi_h;
    int gw = (int)floorf((float)pw * a.group_size / P), gh = (int)floorf((float)ph * a.group_size / P);
    gw = min(max(gw, 0), a.group_size - 1);
    gh = min(max(gh, 0), a.group_size - 1);
    b.chan = (ctop * a.group_size + gh) * a.group_size + gw;
    return b;
}

// sample position -> clamped coordinates; false when the sample lies outside the half-pixel border (kernel.cu:127-132)
__device__ __forceinline__ bool sample_pos(const PoolArgs &a, const Bin &b, int ih, int iw, float &w, float &h) {
    w = b.wstart + iw * b.sub_w;
    h = b.hstart + ih * b.sub_h;
    if (w < -0.5f || w > a.width - 0.5f || h < -0.5f || h > a.height - 0.5f) return false;
    w = fminf(fmaxf(w, 0.f), a.width - 1.f);
    h = fminf(fmaxf(h, 0.f), a.height - 1.f);
    return true;
}

__global__ void deform_psroi_fwd_kernel(PoolArgs a, int64_t count, const float *__restrict__ data, const float *__restrict__ rois,
                                        const float *__restrict__ trans, float *__restrict__ out, float *__restrict__ top_count) {
    for (int64_t index = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; index < count; index += (int64_t)gridDim.x * blockDim.x) {
        const Bin b = bin_geometry(a, rois, trans, index);
        const float *plane = data + ((int64_t)b.batch * a.channels + b.chan) * a.height * a.width;
        float sum = 0.f;
        int cnt = 0;
        for (int ih = 0; ih < a.sample_per_part; ++ih)
            for (int iw = 0; iw < a.sample_per_part; ++iw) {
                float w, h;
                if (!sample_pos(a, b, ih, iw, w, h)) continue;
                const int x1 = (int)floorf(w), x2 = (int)ceilf(w), y1 = (int)floorf(h), y2 = (int)ceilf(h);
                const float dx = w - x1, dy = h - y1;
                sum += (1 - dx) * (1 - dy) * __ldg(plane + y1 * a.width + x1) + (1 - dx) * dy * __ldg(plane + y2 * a.width + x1) +
                       dx * (1 - dy) * __ldg(plane + y1 * a.width + x2) + dx * dy * __ldg(plane + y2 * a.width + x2);
                ++cnt;
            }
        out[index] = cnt == 0 ? 0.f : sum / cnt;
        top_count[index] = (float)cnt;
    }
}

__global__ void deform_psroi_bwd_kernel(PoolArgs a, int64_t count, const float *__restrict__ out_grad,
                                        const float *__restrict__ top_count, const float *__restrict__ data,
                                        const float *__restrict__ rois, const float *__restrict__ trans,
                                        float *__restrict__ in_grad, float *__restrict__ trans_grad) {
    for (int64_t index = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; index < count; index += (int64_t)gridDim.x * blockDim.x) {
        const float cnt = top_count[index];
        if (cnt <= 0.f) continue;
        const Bin b = bin_geometry(a, rois, trans, index);
        const float diff = out_grad[index] / cnt;
        const int64_t base = ((int64_t)b.batch * a.channels + b.chan) * a.height * a.width;
        float gx_acc = 0.f, gy_acc = 0.f;
        for (int ih = 0; ih < a.sample_per_part; ++ih)
            for (int iw = 0; iw < a.sample_per_part; ++iw) {
                float w, h;
                if (!sample_pos(a, b, ih, iw, w, h)) continue;
                const int x0 = (int)floorf(w), x1 = (int)ceilf(w), y0 = (int)floorf(h), y1 = (int)ceilf(h);
                const float dx = w - x0, dy = h - y0;
                atomicAdd(in_grad + base + y0 * a.width + x0, (1 - dx) * (1 - dy) * diff);
                atomicAdd(in_grad + base + y1 * a.width + x0, (1 - dx) * dy * diff);
                atomicAdd(in_grad + base + y0 * a.width + x1, dx * (1 - dy) * diff);
                atomicAdd(in_grad + base + y1 * a.width + x1, dx * dy * diff);
                if (a.no_trans) continue;
                const float u00 = __ldg(data + base + y0 * a.width + x0), u01 = __ldg(data + base + y1 * a.width + x0);
                const float u10 = __ldg(data + base + y0 * a.width + x1), u11 = __ldg(data + base + y1 * a.width + x1);
                gx_acc += (u11 * dy + u10 * (1 - dy) - u01 * dy - u00 * (1 - dy)) * a.trans_std * diff * b.roi_w;
                gy_acc += (u11 * dx + u01 * (1 - dx) - u10 * dx - u00 * (1 - dx)) * a.trans_std * diff * b.roi_h;
            }
        if (!a.no_trans) {          // one atomic per bin and direction instead of one per sample
            atomicAdd(trans_grad + b.tx_index, gx_acc);
            atomicAdd(trans_grad + b.ty_index, gy_acc);
        }
    }
}

int fill_args(PoolArgs &a, int channels, int height, int width, int num_rois, int channels_trans, int no_trans,
              float spatial_scale, int output_dim, int group_size, int pooled, int part_size, int sample_per_part,
              float trans_std) {
    if (channels <= 0 || height <= 0 || width <= 0 || num_rois < 0 || output_dim <= 0 || group_size <= 0 || pooled <= 0 ||
        part_size <= 0 || sample_per_part <= 0)
        return MR_ERR_BAD_SHAPE;
    if (!no_trans && (channels_trans < 2 || channels_trans % 2)) return MR_ERR_BAD_SHAPE;
    if (channels < output_dim * group_size * group_size) return MR_ERR_BAD_SHAPE;     // position-sensitive planes must exist
    a.channels = channels; a.height = height; a.width = width; a.num_rois = num_rois; a.no_trans = no_trans ? 1 : 0;
    a.output_dim = output_dim; a.group_size = group_size; a.pooled = pooled; a.part_size = part_size;
    a.sample_per_part = sample_per_part; a.spatial_scale = spatial_scale; a.trans_std = trans_std;
    a.num_classes = no_trans ? 1 : channels_trans / 2;                                  // kernel.cu:290-291
    a.channels_each_class = no_trans ? output_dim : output_dim / a.num_classes;
    if (a.channels_each_class <= 0) return MR_ERR_BAD_SHAPE;
    return MR_OK;
}

}  // namespace

extern "C" {

int mr_deform_psroi_pool_forward_f32(const float *data, const float *rois, const float *trans, int batch, int channels,
                                     int height, int width, int num_rois, int channels_trans, int no_trans,
                                     float spatial_scale, int output_dim, int group_size, int pooled_size, int part_size,
                                     int sample_per_part, float trans_std, float *out, float *top_count, void *stream) {
    PoolArgs a;
    int rc = fill_args(a, channels, height, width, num_rois, channels_trans, no_trans, spatial_scale, output_dim, group_size,
                       pooled_size, part_size, sample_per_part, trans_std);
    if (rc) return rc;
    (void)batch;
    if (num_rois == 0) return MR_OK;
    if (!data || !rois || !out || !top_count || (!no_trans && !trans)) return MR_ERR_NULL_POINTER;
    const int64_t count = (int64_t)num_rois * output_dim * pooled_size * pooled_size;
    const int blocks = (int)((count + 255) / 256 < mr::sm_count() * 16 ? (count + 255) / 256 : mr::sm_count() * 16);
    deform_psroi_fwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(a, count, data, rois, trans, out, top_count);
    return check_launch("deform_psroi_fwd_kernel");
}

/* in_grad [B,C,H,W] and trans_grad are ACCUMULATED into: zero them first (functions/deform_pool.py:57-59 does). */
int mr_deform_psroi_pool_backward_f32(const float *out_grad, const float *data, const float *rois, const float *trans,
                                      const float *top_count, int batch, int channels, int height, int width, int num_rois,
                                      int channels_trans, int no_trans, float spatial_scale, int output_dim, int group_size,
                                      int pooled_size, int part_size, int sample_per_part, float trans_std, float *in_grad,
                                      float *trans_grad, void *stream) {
    PoolArgs a;
    int rc = fill_args(a, channels, height, width, num_rois, channels_trans, no_trans, spatial_scale, output_dim, group_size,
                       pooled_size, part_size, sample_per_part, trans_std);
    if (rc) return rc;
    (void)batch;
    if (num_rois == 0) return MR_OK;
    if (!out_grad || !data || !rois || !top_count || !in_grad || (!no_trans && (!trans || !trans_grad))) return MR_ERR_NULL_POINTER;
    const int64_t count = (int64_t)num_rois * output_dim * pooled_size * pooled_size;
    const int blocks = (int)((count + 255) / 256 < mr::sm_count() * 16 ? (count + 255) / 256 : mr::sm_count() * 16);
    deform_psroi_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(a, count, out_grad, top_count, data, rois, trans, in_grad, trans_grad);
    return check_launch("deform_psroi_bwd_kernel");
}

}  // extern "C"
