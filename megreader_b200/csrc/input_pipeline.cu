// Recognition input step on the GPU (SURVEY.md section 8 row N3): a ragged batch of decoded HWC images (uint8 straight from
// the decoder, or float32) -> resized, mean-subtracted, scaled, CHW float32 batch [N, 3, dst_h, dst_w] in ONE pass, and the
// ground-truth strings -> padded label matrix.  Replaces, per image on the host, cv2.resize + two numpy passes + a permute
// (data/processes/resize_image.py:29-57, normalize_image.py:10-17) and the python label loop
// (make_recognition_label.py:13-32); shipping uint8 instead of float32 also cuts the host->device bytes by 4.
// HBM-bound and tiny: one thread per output value, arithmetic in input_core.cuh (shared with the CPU harness).
#include "common.cuh"
#include "input_core.cuh"

namespace {
using namespace mr;

template <typename S>
__global__ void resize_normalize_kernel(const S *__restrict__ src, const int64_t *__restrict__ offsets,
                                        const int *__restrict__ heights, const int *__restrict__ widths,
                                        const int *__restrict__ valid_w, int N, int dst_h, int dst_w, double m0, double m1,
                                        double m2, float *__restrict__ out) {
    const int64_t total = (int64_t)N * 3 * dst_h * dst_w;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int n, c, y, x;
        mr_input::decode_index(idx, dst_h, dst_w, n, c, y, x);
        const double mean = c == 0 ? m0 : (c == 1 ? m1 : m2);
        out[idx] = mr_input::resize_normalize_value(src + offsets[n], heights[n], widths[n], dst_h,
                                                    valid_w ? valid_w[n] : dst_w, y, x, c, mean);
    }
}

__global__ void pack_labels_kernel(const unsigned char *__restrict__ text, const int64_t *__restrict__ offsets, int N,
                                   const int *__restrict__ lut, int max_size, int *__restrict__ labels,
                                   int *__restrict__ lengths) {
    const int64_t total = (int64_t)N * max_size;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int n = (int)(idx / max_size), pos = (int)(idx - (int64_t)n * max_size);
        const int len = (int)(offsets[n + 1] - offsets[n]);
        labels[idx] = mr_input::pack_label_value(text + offsets[n], len, pos, lut);
        if (pos == 0) lengths[n] = len < max_size ? len : max_size;
    }
}

int blocks_for(int64_t total) {
    const int64_t b = (total + 255) / 256;
    return (int)(b < 1 ? 1 : (b > mr::sm_count() * 16 ? mr::sm_count() * 16 : b));
}

}  // namespace

extern "C" {

/* src: concatenated HWC 3-channel images (src_is_u8 ? uint8 : float32); offsets[n] = element offset of image n;
 * heights / widths [N] int32; valid_w [N] int32 or NULL (= dst_w: mode "resize"; mode "pad" passes the resized width and the
 * rest of the canvas is zero before normalisation).  All arrays on the device.  out [N,3,dst_h,dst_w] fp32. */
int mr_resize_normalize_f32(const void *src, int src_is_u8, const int64_t *offsets, const int *heights, const int *widths,
                            const int *valid_w, int N, int dst_h, int dst_w, const double *mean3_host, float *out,
                            void *stream) {
    if (N < 0 || dst_h <= 0 || dst_w <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!src || !offsets || !heights || !widths || !mean3_host || !out) return MR_ERR_NULL_POINTER;
    const int64_t total = (int64_t)N * 3 * dst_h * dst_w;
    cudaStream_t st = (cudaStream_t)stream;
    if (src_is_u8)
        resize_normalize_kernel<unsigned char><<<blocks_for(total), 256, 0, st>>>((const unsigned char *)src, offsets, heights, widths, valid_w, N, dst_h,
                                                                                  dst_w, mean3_host[0], mean3_host[1], mean3_host[2], out);
    else
        resize_normalize_kernel<float><<<blocks_for(total), 256, 0, st>>>((const float *)src, offsets, heights, widths, valid_w, N, dst_h, dst_w,
                                                                          mean3_host[0], mean3_host[1], mean3_host[2], out);
    return check_launch("resize_normalize_kernel");
}

/* text: concatenated label bytes; offsets [N+1] int64; lut [256] int32 (byte -> class index); labels [N,max_size] int32,
 * lengths [N] int32.  All on the device. */
int mr_pack_labels(const unsigned char *text, const int64_t *offsets, int N, const int *lut, int max_size, int *labels,
                   int *lengths, void *stream) {
    if (N < 0 || max_size <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!offsets || !lut || !labels || !lengths) return MR_ERR_NULL_POINTER;
    pack_labels_kernel<<<blocks_for((int64_t)N * max_size), 256, 0, (cudaStream_t)stream>>>(text, offsets, N, lut, max_size, labels, lengths);
    return check_launch("pack_labels_kernel");
}

}  // extern "C"
