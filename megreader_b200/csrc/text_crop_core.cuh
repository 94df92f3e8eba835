// Per-quad and per-pixel arithmetic of ImageCropper.crop (data/crop_file_dataset.py:85-124 with concern/cv.py:5-12), shared by
// the CUDA kernels (text_crop.cu) and by a host harness (tests/host_harness/text_crop_core_host.cpp) built with
// -ffp-contract=off, so the device and the host round every product and sum alike (fmul / fadd / dmul of db_boxes_core).
//
// Per quad (setup):  cv2.minAreaRect of the float32 corners (db_boxes_core's hull and calipers), the reference's angle rule
//                    (< -45: +180, else swap the sides and +90), cv2.boxPoints; the sides w = |p1 - p0|, h = |p2 - p1| as
//                    np.linalg.norm gives them in float32; cv2.getPerspectiveTransform(box, [(0,0),(w,0),(w,h),(0,h)]) (its
//                    8 x 8 system solved by cv2's LU with partial pivoting) and the inverse cv2.warpPerspective applies;
//                    the crop size (int(w), int(h)) -- cv2 takes the source's size when either side is 0 -- and the turn
//                    of ensure_horizontal (h > 1.5 w on the integer size).
// Per output pixel:  ResizeImage ("resize" or "pad", INTER_LINEAR as input_core.cuh restates it) of the possibly turned crop,
//                    each of its four taps one cv2.warpPerspective INTER_LINEAR sample of the source (cv2's per-pixel W,
//                    INTER_TAB_SIZE = 32 source coordinates, its integer bilinear table for uint8 with the rounding to uint8,
//                    its float table for float32), then NormalizeImage.  The crop itself is never stored.
#pragma once
#include "db_boxes_core.cuh"
#include "input_core.cuh"

namespace mr_textcrop {

using mr_dbbox::dadd;
using mr_dbbox::dmul;
using mr_dbbox::dsub;
using mr_dbbox::fadd;
using mr_dbbox::fmul;
using mr_dbbox::fsub;

// per-image status bits
enum Status { kBadShape = 1, kBadPixels = 2, kBadCount = 4, kOverflow = 8, kZeroSide = 16, kCropTooLarge = 32 };

constexpr int kMaxSide = 32766;          // cv2's remap refuses images and maps with a side of SHRT_MAX or more

#ifdef __CUDA_ARCH__
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float fsqrt(float a) { return __fsqrt_rn(a); }
#else
inline double ddiv(double a, double b) { return a / b; }
inline float fsqrt(float a) { return sqrtf(a); }
#endif

struct Crop {
    double P[9];                         // getPerspectiveTransform: box corners -> crop
    double M[9];                         // its inverse as warpPerspective computes it: crop pixel -> source
    float box[8];                        // min_area_rect's corners
    float w, h;                          // the float32 sides
    int cw, ch;                          // the warp's output size (the source's when int(w) or int(h) is 0)
    int bw;                              // warpPerspective's block width for that size
    int turned;                          // ensure_horizontal turned the crop
    int rh, rw;                          // the resize input: the crop, turned or not
    int valid_w;                         // the resized width ("pad": at most out_w, the rest of the canvas is zero)
    int flags;                           // kZeroSide, kCropTooLarge
};

// concern/cv.py's min_area_rect: cv2.minAreaRect of the float32 quad q[8], the angle rule, cv2.boxPoints -> box[8]
__host__ __device__ inline void min_area_rect(const float *q, float *box) {
    mr_dbbox::PtT<float> p[4];
    for (int i = 0; i < 4; ++i) p[i] = mr_dbbox::PtT<float>{q[2 * i], q[2 * i + 1]};
    int o[4], stack[6], hull[4];
    const int k = mr_dbbox::convex_hull(p, 4, o, stack, hull);
    float qx[4], qy[4], vx[4], vy[4], inv[4];
    for (int j = 0; j < k; ++j) { qx[j] = p[hull[j]].x; qy[j] = p[hull[j]].y; }
    mr_dbbox::Rect r = mr_dbbox::min_area_rect_hull(qx, qy, k, vx, vy, inv);
    if (r.angle < -45.f) {
        r.angle = (float)dadd((double)r.angle, 180.);
    } else {
        const float t = r.w; r.w = r.h; r.h = t;
        r.angle = (float)dadd((double)r.angle, 90.);
    }
    float px[4], py[4];
    mr_dbbox::box_points(r, px, py);
    for (int i = 0; i < 4; ++i) { box[2 * i] = px[i]; box[2 * i + 1] = py[i]; }
}

// np.linalg.norm of the float32 difference of two corners: the float32 dot product, then its float32 square root
__host__ __device__ inline float side(const float *a, const float *b) {
    const float dx = fsub(b[0], a[0]), dy = fsub(b[1], a[1]);
    return fsqrt(fadd(fmul(dx, dx), fmul(dy, dy)));
}

// cv::solve(A, b, x, DECOMP_LU) for 8 x 8: LUImpl<double> (partial pivoting, eps = 100 DBL_EPSILON) with cv2's order of
// operations; a singular system gives x = 0.  Overwrites a and b; the solution is left in b.
__host__ __device__ inline bool lu_solve8(double (*a)[8], double *b) {
    const double eps = 2.220446049250313080847e-16 * 100;
    for (int i = 0; i < 8; ++i) {
        int k = i;
        for (int j = i + 1; j < 8; ++j)
            if (fabs(a[j][i]) > fabs(a[k][i])) k = j;
        if (fabs(a[k][i]) < eps) {
            for (int j = 0; j < 8; ++j) b[j] = 0.;
            return false;
        }
        if (k != i) {
            for (int j = i; j < 8; ++j) { const double t = a[i][j]; a[i][j] = a[k][j]; a[k][j] = t; }
            const double t = b[i]; b[i] = b[k]; b[k] = t;
        }
        const double d = ddiv(-1., a[i][i]);
        for (int j = i + 1; j < 8; ++j) {
            const double alpha = dmul(a[j][i], d);
            for (int c = i + 1; c < 8; ++c) a[j][c] = dadd(a[j][c], dmul(alpha, a[i][c]));
            b[j] = dadd(b[j], dmul(alpha, b[i]));
        }
    }
    for (int i = 7; i >= 0; --i) {
        double s = b[i];
        for (int c = i + 1; c < 8; ++c) s = dsub(s, dmul(a[i][c], b[c]));
        b[i] = ddiv(s, a[i][i]);
    }
    return true;
}

// cv2.getPerspectiveTransform(src, dst) (float32 corners, x / y interleaved): the rows' products -src * dst in float32
__host__ __device__ inline void perspective_transform(const float *src, const float *dst, double *P) {
    double a[8][8], b[8];
    for (int i = 0; i < 4; ++i) {
        const float sx = src[2 * i], sy = src[2 * i + 1], dx = dst[2 * i], dy = dst[2 * i + 1];
        a[i][0] = a[i + 4][3] = sx;
        a[i][1] = a[i + 4][4] = sy;
        a[i][2] = a[i + 4][5] = 1.;
        a[i][3] = a[i][4] = a[i][5] = a[i + 4][0] = a[i + 4][1] = a[i + 4][2] = 0.;
        a[i][6] = fmul(-sx, dx);
        a[i][7] = fmul(-sy, dx);
        a[i + 4][6] = fmul(-sx, dy);
        a[i + 4][7] = fmul(-sy, dy);
        b[i] = dx;
        b[i + 4] = dy;
    }
    lu_solve8(a, b);
    for (int i = 0; i < 8; ++i) P[i] = b[i];
    P[8] = 1.;
}

// cv::invert(P, M, DECOMP_LU) of a 3 x 3 double matrix: the adjugate over the cofactor determinant; zero when it is 0
__host__ __device__ inline void invert3(const double *m, double *r) {
    auto cof = [](double a, double b, double c, double d) { return dsub(dmul(a, b), dmul(c, d)); };
    const double det = dadd(dsub(dmul(m[0], cof(m[4], m[8], m[5], m[7])), dmul(m[1], cof(m[3], m[8], m[5], m[6]))),
                            dmul(m[2], cof(m[3], m[7], m[4], m[6])));
    if (det == 0.) {
        for (int i = 0; i < 9; ++i) r[i] = 0.;
        return;
    }
    const double d = ddiv(1., det);
    r[0] = dmul(cof(m[4], m[8], m[5], m[7]), d);
    r[1] = dmul(cof(m[2], m[7], m[1], m[8]), d);
    r[2] = dmul(cof(m[1], m[5], m[2], m[4]), d);
    r[3] = dmul(cof(m[5], m[6], m[3], m[8]), d);
    r[4] = dmul(cof(m[0], m[8], m[2], m[6]), d);
    r[5] = dmul(cof(m[2], m[3], m[0], m[5]), d);
    r[6] = dmul(cof(m[3], m[7], m[4], m[6]), d);
    r[7] = dmul(cof(m[1], m[6], m[0], m[7]), d);
    r[8] = dmul(cof(m[0], m[4], m[1], m[3]), d);
}

// warpPerspective works in blocks of at most 32 x 32 output pixels; its x coordinate is the block's origin plus the offset in
// the block, so the block width is part of the arithmetic
__host__ __device__ inline int warp_block_width(int cw, int ch) {
    const int bh0 = ch < 16 ? ch : 16;
    return 1024 / bh0 < cw ? 1024 / bh0 : cw;
}

// ResizeImage's width for an rh x rw input (resize_image.py:41-48): mode 0 "resize" -> out_w, mode 1 "pad" ->
// min(out_w, max(int(out_h / rh * rw / 32 + 0.5) * 32, 32)) in Python's double arithmetic
__host__ __device__ inline int resized_width(int mode, int out_h, int out_w, int rh, int rw) {
    if (mode == 0) return out_w;
    const int w = (int)dadd(ddiv(dmul(ddiv((double)out_h, (double)rh), (double)rw), 32.), 0.5) * 32;
    const int v = w > 32 ? w : 32;
    return v < out_w ? v : out_w;
}

// Everything ImageCropper.crop derives from the quad q[8] (float32 corners) for an img_h x img_w source
__host__ __device__ inline void setup(const float *q, int img_h, int img_w, int mode, int out_h, int out_w, Crop &c) {
    min_area_rect(q, c.box);
    c.w = side(c.box, c.box + 2);
    c.h = side(c.box + 2, c.box + 4);
    const float dst[8] = {0.f, 0.f, c.w, 0.f, c.w, c.h, 0.f, c.h};
    perspective_transform(c.box, dst, c.P);
    invert3(c.P, c.M);
    // (int(w), int(h)): truncation; cv2 takes the source's size for an empty dsize
    const float lim = 2147483520.f;
    c.cw = (int)(c.w < lim ? c.w : lim);
    c.ch = (int)(c.h < lim ? c.h : lim);
    c.flags = 0;
    if (c.cw <= 0 || c.ch <= 0) {
        c.cw = img_w;
        c.ch = img_h;
        c.flags |= kZeroSide;
    }
    if (c.cw > kMaxSide || c.ch > kMaxSide) c.flags |= kCropTooLarge;
    c.bw = warp_block_width(c.cw, c.ch);
    c.turned = (double)c.ch > dmul((double)c.cw, 1.5);
    c.rh = c.turned ? c.cw : c.ch;
    c.rw = c.turned ? c.ch : c.cw;
    c.valid_w = resized_width(mode, out_h, out_w, c.rh, c.rw);
}

template <typename S> __host__ __device__ inline float px(const S *img, int w, int y, int x, int c) {
    return (float)img[((int64_t)y * w + x) * 3 + c];
}

__host__ __device__ inline int clamp_short(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }

// cv2.warpPerspective(img, P, (cw, ch), INTER_LINEAR, BORDER_CONSTANT, 0) at crop pixel (xd, yd), three channels, as float32
// (a uint8 source's value is the uint8 the warp stores).  Taps outside the source are 0.
template <typename S>
__host__ __device__ inline void warp_sample(const S *img, int h, int w, const Crop &c, int xd, int yd, float *out) {
    const double *M = c.M;
    const int xb = xd / c.bw * c.bw, x1 = xd - xb;
    const double X0 = dadd(dadd(dmul(M[0], (double)xb), dmul(M[1], (double)yd)), M[2]);
    const double Y0 = dadd(dadd(dmul(M[3], (double)xb), dmul(M[4], (double)yd)), M[5]);
    const double W0 = dadd(dadd(dmul(M[6], (double)xb), dmul(M[7], (double)yd)), M[8]);
    double W = dadd(W0, dmul(M[6], (double)x1));
    W = W != 0. ? ddiv(32., W) : 0.;
    // std::max(INT_MIN, std::min(INT_MAX, v)), which maps NaN to INT_MAX, then cvRound (half to even)
    double fX = dmul(dadd(X0, dmul(M[0], (double)x1)), W), fY = dmul(dadd(Y0, dmul(M[3], (double)x1)), W);
    fX = fX < 2147483647. ? fX : 2147483647.;
    fY = fY < 2147483647. ? fY : 2147483647.;
    fX = -2147483648. < fX ? fX : -2147483648.;
    fY = -2147483648. < fY ? fY : -2147483648.;
    const int X = (int)rint(fX), Y = (int)rint(fY);
    const int sx = clamp_short(X >> 5), sy = clamp_short(Y >> 5), ax = X & 31, ay = Y & 31;
    const bool in_x0 = sx >= 0 && sx < w, in_x1 = sx + 1 >= 0 && sx + 1 < w;
    const bool in_y0 = sy >= 0 && sy < h, in_y1 = sy + 1 >= 0 && sy + 1 < h;
    const bool u8 = sizeof(S) == 1;
    for (int k = 0; k < 3; ++k) {
        const float v00 = in_y0 && in_x0 ? px(img, w, sy, sx, k) : 0.f, v01 = in_y0 && in_x1 ? px(img, w, sy, sx + 1, k) : 0.f;
        const float v10 = in_y1 && in_x0 ? px(img, w, sy + 1, sx, k) : 0.f, v11 = in_y1 && in_x1 ? px(img, w, sy + 1, sx + 1, k) : 0.f;
        if (u8) {                        // BilinearTab_i: 32 (32 - ay)(32 - ax) ... in 1 << 15, then FixedPtCast
            const int s = (int)v00 * (32 * (32 - ay) * (32 - ax)) + (int)v01 * (32 * (32 - ay) * ax) +
                          (int)v10 * (32 * ay * (32 - ax)) + (int)v11 * (32 * ay * ax);
            const int r = (s + (1 << 14)) >> 15;
            out[k] = (float)(r < 0 ? 0 : (r > 255 ? 255 : r));
        } else {                         // BilinearTab_f, summed left to right
            const float fx = fmul((float)ax, 1.f / 32.f), fy = fmul((float)ay, 1.f / 32.f);
            const float gx = fsub(1.f, fx), gy = fsub(1.f, fy);
            out[k] = fadd(fadd(fadd(fmul(v00, fmul(gy, gx)), fmul(v01, fmul(gy, fx))), fmul(v10, fmul(fy, gx))), fmul(v11, fmul(fy, fx)));
        }
    }
}

// The value of the resize input (the crop, turned by ensure_horizontal: np.flip(np.swapaxes(crop, 0, 1), 0)) at (r, col)
template <typename S>
__host__ __device__ inline void turned_sample(const S *img, int h, int w, const Crop &c, int r, int col, float *out) {
    if (c.turned) warp_sample(img, h, w, c, c.cw - 1 - r, col, out);
    else warp_sample(img, h, w, c, col, r, out);
}

// The normalised output pixel (y, x) of the [out_h, out_w] canvas, three channels: ResizeImage of the turned crop (columns
// >= valid_w are the zero padding of "pad"), then (v - mean) / 255.  A crop cv2 would refuse gives the zero canvas.
template <typename S>
__host__ __device__ inline void output_pixel(const Crop &c, const S *img, int h, int w, int out_h, const double *mean, int y, int x,
                                             float *out) {
    float v[3] = {0.f, 0.f, 0.f};
    if (x < c.valid_w && !(c.flags & kCropTooLarge)) {
        const mr_input::Axis lx = mr_input::axis_taps(x, c.valid_w, c.rw, true), ly = mr_input::axis_taps(y, out_h, c.rh, false);
        float t00[3], t01[3], t10[3], t11[3];
        turned_sample(img, h, w, c, ly.i0, lx.i0, t00);
        turned_sample(img, h, w, c, ly.i0, lx.i1, t01);
        turned_sample(img, h, w, c, ly.i1, lx.i0, t10);
        turned_sample(img, h, w, c, ly.i1, lx.i1, t11);
        for (int k = 0; k < 3; ++k) {
            const float r0 = fadd(fmul(t00[k], lx.w0), fmul(t01[k], lx.w1));
            const float r1 = fadd(fmul(t10[k], lx.w0), fmul(t11[k], lx.w1));
            v[k] = fadd(fmul(r0, ly.w0), fmul(r1, ly.w1));
        }
    }
    for (int k = 0; k < 3; ++k) out[k] = mr_input::normalize_value(v[k], mean[k]);
}

}  // namespace mr_textcrop
