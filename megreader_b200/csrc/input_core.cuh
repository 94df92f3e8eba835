// Per-pixel arithmetic of the recognition input step (SURVEY.md section 8 row N3), shared by the CUDA kernel
// (input_pipeline.cu) and by a host-side harness (tests/host_harness/input_core_host.cpp) that runs the SAME routine on the
// CPU against the oracle -- so that only the launch glue is specific to the device build.
//
//   cv2.resize(float32 HWC, (dst_w, dst_h))  [INTER_LINEAR, OpenCV resize.cpp: half-pixel centres, scale = 1/(dst/src) in
//   double, fraction stored as float, left/right neighbour clamped by zeroing the fraction, rows clamped by index]
//   -> image -= RGB_MEAN (float64 vector, result stored as float32) ; image /= 255.f   (normalize_image.py:13-14)
//   -> HWC -> CHW                                                                       (normalize_image.py:15)
#pragma once
#include <math.h>
#include <stdint.h>

#if !defined(__CUDACC__) && !defined(__host__)
#define __host__
#define __device__
#endif

namespace mr_input {

struct Axis { int i0, i1; float w0, w1; };

// (d + 0.5) * scale - 0.5 in double with both roundings, as cv2's x86 build computes it (no fused multiply-add on the device)
__host__ __device__ inline double src_coord(int d, double scale) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
#else
    return ((double)d + 0.5) * scale - 0.5;
#endif
}

// source taps of destination index d along an axis of `src` samples resized to `dst` samples
__host__ __device__ inline Axis axis_taps(int d, int dst, int src, bool zero_fraction_at_border) {
    const double scale = 1.0 / ((double)dst / (double)src);
    float f = (float)src_coord(d, scale);
    int s = (int)floorf(f);
    f -= (float)s;
    Axis a;
    if (zero_fraction_at_border) {                 // horizontal rule: fraction forced to 0 at either end
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
        a.i0 = s;
        a.i1 = s + 1 < src ? s + 1 : src - 1;
    } else {                                       // vertical rule: both row indices clamped, fraction kept
        a.i0 = s < 0 ? 0 : (s > src - 1 ? src - 1 : s);
        a.i1 = s + 1 < 0 ? 0 : (s + 1 > src - 1 ? src - 1 : s + 1);
    }
    a.w0 = 1.f - f;
    a.w1 = f;
    return a;
}

template <typename S> __host__ __device__ inline float src_value(const S *img, int W, int y, int x, int c) {
    return (float)img[((int64_t)y * W + x) * 3 + c];
}

// NormalizeImage of one value: float32 array minus float64 vector, stored as float32, then / 255
__host__ __device__ inline float normalize_value(float v, double mean_c) {
    const float centred = (float)((double)v - mean_c);
    return centred / 255.f;
}

// one output value: destination pixel (y, x), channel c of an image resized to [dst_h, valid_w] and placed at the left of a
// [dst_h, dst_w] canvas (columns >= valid_w are the zero padding of mode "pad"), then normalised
template <typename S>
__host__ __device__ inline float resize_normalize_value(const S *img, int H, int W, int dst_h, int valid_w, int y, int x, int c,
                                                        double mean_c) {
    float v = 0.f;
    if (x < valid_w) {
        const Axis ax = axis_taps(x, valid_w, W, true), ay = axis_taps(y, dst_h, H, false);
        const float r0 = src_value(img, W, ay.i0, ax.i0, c) * ax.w0 + src_value(img, W, ay.i0, ax.i1, c) * ax.w1;
        const float r1 = src_value(img, W, ay.i1, ax.i0, c) * ax.w0 + src_value(img, W, ay.i1, ax.i1, c) * ax.w1;
        v = r0 * ay.w0 + r1 * ay.w1;
    }
    return normalize_value(v, mean_c);
}

// flat output index of [N, 3, dst_h, dst_w] -> (n, c, y, x)
__host__ __device__ inline void decode_index(int64_t idx, int dst_h, int dst_w, int &n, int &c, int &y, int &x) {
    x = (int)(idx % dst_w);
    y = (int)((idx / dst_w) % dst_h);
    c = (int)((idx / dst_w / dst_h) % 3);
    n = (int)(idx / dst_w / dst_h / 3);
}

// label packing (concern/charsets.py:52-58 + make_recognition_label.py:22-31): byte string -> class indices through a
// 256-entry table, zero (blank) padded / truncated to max_size; length = min(len, max_size)
__host__ __device__ inline int pack_label_value(const unsigned char *text, int len, int pos, const int *lut) {
    return pos < len ? lut[text[pos]] : 0;
}

}  // namespace mr_input
