// Per-image and per-pixel arithmetic of the DB detector's input batch (seg_detector_db.yaml's data processes before the
// targets), shared by the CUDA kernels (db_batch.cu) and by a host harness (tests/host_harness/db_batch_core_host.cpp) built
// with -ffp-contract=off, so the device and the host round every product and sum alike (fmul / fadd / dmul of db_boxes_core).
//
// Training:  AugmentDetectionData: imgaug Sequential([Fliplr(p), Affine(rotate=(lo, hi)), Resize((lo, hi))]) restated after
//            imgaug 0.4.0 with its cv2 backend (DESIGN §7) -> RandomCropData(size, max_tries, min_crop_side_ratio)
//            (data/processes/random_crop_data.py) -> MakeICDARData -> NormalizeImage.
// Validation: AugmentDetectionData([Resize({width, height})]) -> MakeICDARData -> NormalizeImage.
//
// The pixels are never materialised at the resized size: the kernels keep the flipped and rotated image (cv2.warpAffine,
// INTER_LINEAR, constant 0 border) and evaluate, per output pixel, cv2.resize's INTER_CUBIC at the four INTER_LINEAR taps of
// the crop's resize (input_core.cuh), then NormalizeImage.
#pragma once
#include "db_boxes_core.cuh"
#include "input_core.cuh"

namespace mr_dbbatch {

using mr_dbbox::dadd;
using mr_dbbox::dmul;
using mr_dbbox::dsub;
using mr_dbbox::fadd;
using mr_dbbox::fmul;
using mr_dbbox::fsub;

constexpr double kMaxScale = 4.0;        // largest Resize scale the workspace is sized for

enum Status { kBadShape = 1, kBadPixels = 2, kBadOffsets = 4 };

struct Params {
    int mode;                            // 0 training, 1 validation
    int out_h, out_w;                    // training: RandomCropData's canvas (size[1], size[0]); validation: the Resize target
    int max_tries;
    double min_ratio, flip_p, rot_lo, rot_hi, scale_lo, scale_hi;
    double mean[3];
};

// Draws per image: flip, angle, scale, then for each of crop_area's two rounds and each try the two x and the two y draws of
// np.random.choice(axis, size=2)
__host__ __device__ inline int draws_needed(int max_tries) { return 3 + 8 * max_tries; }

struct Geom {
    int h, w;                            // input (the `shape` AugmentData records)
    int hs, ws;                          // after Resize
    int flip;
    double M[6];                         // Affine's forward matrix (keypoints)
    double A[6];                         // its inverse as cv2.warpAffine computes it (pixels)
    int cx, cy, cw, ch;                  // the crop in the resized image
    int oh, ow;                          // the crop's size on the canvas
    double scale;
    int status;
};

__host__ __device__ inline int imin(int a, int b) { return a < b ? a : b; }
__host__ __device__ inline int imax(int a, int b) { return a > b ? a : b; }
__host__ __device__ inline int iclamp(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
__host__ __device__ inline int cv_round(double v) { return (int)rint(v); }   // cvRound / np.round: half to even

// sin and cos by their Taylor series in Horner form with explicitly rounded operations: the same bits on the host and the
// device (libm's and CUDA's cos may differ in the last place).  Within 1e-15 of the true values for |r| <= pi.
__host__ __device__ inline void sin_cos(double r, double &s, double &c) {
    const double r2 = dmul(r, r);
    double ps = 1., pc = 1.;
    for (int k = 16; k >= 1; --k) {
        ps = dsub(1., dmul(dmul(r2, ps), 1. / ((2. * k) * (2. * k + 1.))));
        pc = dsub(1., dmul(dmul(r2, pc), 1. / ((2. * k - 1.) * (2. * k))));
    }
    s = dmul(r, ps);
    c = pc;
}

// imgaug's Affine(rotate=deg) of a w x h image: translate the centre (w / 2 - 0.5, h / 2 - 0.5) to the origin, rotate by
// deg (skimage's AffineTransform(rotation)), translate back.  M maps input to output coordinates.
__host__ __device__ inline void rotation_matrix(double deg, int w, int h, double *M) {
    double s, c;
    sin_cos(dmul(deg, 3.14159265358979323846 / 180.), s, c);
    const double cx = dsub((double)w / 2., 0.5), cy = dsub((double)h / 2., 0.5);
    M[0] = c; M[1] = -s; M[2] = dadd(dsub(cx, dmul(c, cx)), dmul(s, cy));
    M[3] = s; M[4] = c;  M[5] = dsub(dsub(cy, dmul(s, cx)), dmul(c, cy));
}

// cv::warpAffine's inversion of a forward matrix (imgwarp.cpp, without WARP_INVERSE_MAP)
__host__ __device__ inline void invert_affine(const double *M, double *A) {
    double D = dsub(dmul(M[0], M[4]), dmul(M[1], M[3]));
    D = D != 0. ? 1. / D : 0.;
    A[0] = dmul(M[4], D); A[1] = dmul(M[1], -D); A[3] = dmul(M[3], -D); A[4] = dmul(M[0], D);
    A[2] = dsub(dmul(-A[0], M[2]), dmul(A[1], M[5]));
    A[5] = dsub(dmul(-A[3], M[2]), dmul(A[4], M[5]));
}

// The augmentation of one h x w image from its draws u[0..3): flip when u0 < p, angle lo + u1 (hi - lo), scale
// lo + u2 (hi - lo) for both sides with the new sides round(side * scale) (Python's round: half to even), at least 1.
// Validation: no flip, no rotation, the new sides are the Resize target.
__host__ __device__ inline void augment_geometry(const Params &P, const float *u, int h, int w, Geom &g) {
    g.h = h; g.w = w;
    g.flip = 0;
    double deg = 0.;
    if (P.mode == 0) {
        g.flip = (double)u[0] < P.flip_p;
        deg = dadd(P.rot_lo, dmul((double)u[1], dsub(P.rot_hi, P.rot_lo)));
        const double s = dadd(P.scale_lo, dmul((double)u[2], dsub(P.scale_hi, P.scale_lo)));
        g.hs = imax(1, cv_round(dmul(s, (double)h)));
        g.ws = imax(1, cv_round(dmul(s, (double)w)));
    } else {
        g.hs = P.out_h;
        g.ws = P.out_w;
    }
    rotation_matrix(deg, w, h, g.M);
    invert_affine(g.M, g.A);
    g.cx = g.cy = 0; g.cw = g.ws; g.ch = g.hs;
    g.oh = g.hs; g.ow = g.ws;
    g.scale = 1.;
    g.status = 0;
}

// A keypoint through the flip (x -> w - x), the rotation and the resize ((x / w) * new_w), in float64
__host__ __device__ inline void augment_point(const Geom &g, double x, double y, double &ox, double &oy) {
    if (g.flip) x = dsub((double)g.w, x);
    const double rx = dadd(dadd(dmul(g.M[0], x), dmul(g.M[1], y)), g.M[2]);
    const double ry = dadd(dadd(dmul(g.M[3], x), dmul(g.M[4], y)), g.M[5]);
    ox = dmul(rx / (double)g.w, (double)g.ws);
    oy = dmul(ry / (double)g.h, (double)g.hs);
}

// ---- RandomCropData.crop_area ----

// The slice [a:b] of a length-L array as Python resolves it: negative bounds count from the end, large ones are clipped
__host__ __device__ inline void py_slice(int a, int b, int L, int &lo, int &hi) {
    lo = a < 0 ? imax(a + L, 0) : imin(a, L);
    hi = b < 0 ? imax(b + L, 0) : imin(b, L);
    if (hi < lo) hi = lo;
}

// The slices crop_area marks for one quad q[8] (x0, y0, ..., float64): np.round(points).astype(np.int32), then
// w_array[minx:maxx] and h_array[miny:maxy]
__host__ __device__ inline void marked_slices(const double *q, int ws, int hs, int &x0, int &x1, int &y0, int &y1) {
    int minx = cv_round(q[0]), maxx = minx, miny = cv_round(q[1]), maxy = miny;
    for (int k = 1; k < 4; ++k) {
        const int x = cv_round(q[2 * k]), y = cv_round(q[2 * k + 1]);
        minx = imin(minx, x); maxx = imax(maxx, x);
        miny = imin(miny, y); maxy = imax(maxy, y);
    }
    py_slice(minx, maxx, ws, x0, x1);
    py_slice(miny, maxy, hs, y0, y1);
}

// RandomCropData.is_poly_outside_rect on the unrounded corners
__host__ __device__ inline bool poly_outside_rect(const double *q, double x, double y, double w, double h) {
    double x0 = q[0], x1 = q[0], y0 = q[1], y1 = q[1];
    for (int k = 1; k < 4; ++k) {
        x0 = fmin(x0, q[2 * k]); x1 = fmax(x1, q[2 * k]);
        y0 = fmin(y0, q[2 * k + 1]); y1 = fmax(y1, q[2 * k + 1]);
    }
    if (x1 < x || x0 > dadd(x, w)) return true;
    if (y1 < y || y0 > dadd(y, h)) return true;
    return false;
}

// One of np.random.choice(axis)'s picks from the draw u: axis[min(floor(u * len), len - 1)]
__host__ __device__ inline int pick(const int *axis, int len, float u) {
    return axis[iclamp((int)floor(dmul((double)u, (double)len)), 0, len - 1)];
}

// One call of crop_area after the axes are built: max_tries tries from the draws u[4 * max_tries] (x, x, y, y per try).
// fixed: the first call, with `size` (the crop's height also comes from the width).  The overlap test stops at the first care
// polygon (tags[p] == 0) of polys[k][8] that is not outside.
__host__ __device__ inline bool crop_round(const Params &P, const float *u, bool fixed, int ws, int hs, const int *w_axis, int nw,
                                           const int *h_axis, int nh, const double *polys, const unsigned char *tags, int k,
                                           int &cx, int &cy, int &cw, int &ch) {
    for (int t = 0; t < P.max_tries; ++t) {
        const float *d = u + 4 * t;
        const int xa = pick(w_axis, nw, d[0]), xb = pick(w_axis, nw, d[1]);
        int xmin = imin(xa, xb), xmax = fixed ? xmin + P.out_w : imax(xa, xb);
        xmin = iclamp(xmin, 0, ws - 1);
        xmax = iclamp(xmax, 0, ws - 1);
        const int ya = pick(h_axis, nh, d[2]), yb = pick(h_axis, nh, d[3]);
        int ymin = imin(ya, yb), ymax = fixed ? ymin + P.out_w : imax(ya, yb);
        ymin = iclamp(ymin, 0, hs - 1);
        ymax = iclamp(ymax, 0, hs - 1);
        if ((double)(xmax - xmin) < dmul(P.min_ratio, (double)ws) || (double)(ymax - ymin) < dmul(P.min_ratio, (double)hs)) continue;
        for (int p = 0; p < k; ++p) {
            if (tags[p]) continue;
            if (!poly_outside_rect(polys + 8 * p, xmin, ymin, xmax - xmin, ymax - ymin)) {
                cx = xmin; cy = ymin; cw = xmax - xmin; ch = ymax - ymin;
                return true;
            }
        }
    }
    return false;
}

// crop_area from the built axes (the indices of w_array / h_array still 0), then the canvas scale and size:
// scale = min(size_w / cw, size_h / ch); h = int(ch * scale), w = int(cw * scale)
__host__ __device__ inline void choose_crop(const Params &P, const float *u, const int *w_axis, int nw, const int *h_axis, int nh,
                                            const double *polys, const unsigned char *tags, int k, Geom &g) {
    g.cx = g.cy = 0; g.cw = g.ws; g.ch = g.hs;
    if (nw > 0 && nh > 0 &&
        !crop_round(P, u + 3, true, g.ws, g.hs, w_axis, nw, h_axis, nh, polys, tags, k, g.cx, g.cy, g.cw, g.ch))
        crop_round(P, u + 3 + 4 * P.max_tries, false, g.ws, g.hs, w_axis, nw, h_axis, nh, polys, tags, k, g.cx, g.cy, g.cw, g.ch);
    const double sw = (double)P.out_w / (double)g.cw, sh = (double)P.out_h / (double)g.ch;
    g.scale = sw < sh ? sw : sh;
    g.oh = (int)dmul((double)g.ch, g.scale);
    g.ow = (int)dmul((double)g.cw, g.scale);
}

// A polygon's corner on the canvas: (point - (cx, cy)) * scale, float64
__host__ __device__ inline double crop_coord(double v, int origin, double scale) { return dmul(dsub(v, (double)origin), scale); }

// ---- pixels ----

template <typename S> __host__ __device__ inline float px(const S *img, int w, int y, int x, int c) {
    return (float)img[((int64_t)y * w + x) * 3 + c];
}

// cv2.warpAffine(flip(img), M, (w, h), INTER_LINEAR, BORDER_CONSTANT, 0) at output pixel (y, x), three channels: cv2's
// fixed-point source coordinates (AB_BITS = 10, rounded to 1/32) and its float bilinear table, summed left to right.  The
// flip is folded into the source column.
template <typename S>
__host__ __device__ inline void warp_pixel(const S *img, int h, int w, bool flip, const double *A, int y, int x, float *out) {
    const int X0 = cv_round(dmul(dadd(dmul(A[1], (double)y), A[2]), 1024.)) + 16;
    const int Y0 = cv_round(dmul(dadd(dmul(A[4], (double)y), A[5]), 1024.)) + 16;
    const int X = (X0 + cv_round(dmul(dmul(A[0], (double)x), 1024.))) >> 5;
    const int Y = (Y0 + cv_round(dmul(dmul(A[3], (double)x), 1024.))) >> 5;
    const int sx = X >> 5, sy = Y >> 5;
    const float ax = fmul((float)(X & 31), 1.f / 32.f), ay = fmul((float)(Y & 31), 1.f / 32.f);
    const float wx0 = fsub(1.f, ax), wy0 = fsub(1.f, ay);
    const float wt[4] = {fmul(wy0, wx0), fmul(wy0, ax), fmul(ay, wx0), fmul(ay, ax)};
    const bool in_x0 = sx >= 0 && sx < w, in_x1 = sx + 1 >= 0 && sx + 1 < w;
    const bool in_y0 = sy >= 0 && sy < h, in_y1 = sy + 1 >= 0 && sy + 1 < h;
    const int c0 = flip ? w - 1 - sx : sx, c1 = flip ? w - 2 - sx : sx + 1;
    for (int c = 0; c < 3; ++c) {
        const float v00 = in_y0 && in_x0 ? px(img, w, sy, c0, c) : 0.f, v01 = in_y0 && in_x1 ? px(img, w, sy, c1, c) : 0.f;
        const float v10 = in_y1 && in_x0 ? px(img, w, sy + 1, c0, c) : 0.f, v11 = in_y1 && in_x1 ? px(img, w, sy + 1, c1, c) : 0.f;
        out[c] = fadd(fadd(fadd(fmul(v00, wt[0]), fmul(v01, wt[1])), fmul(v10, wt[2])), fmul(v11, wt[3]));
    }
}

// cv2's interpolateCubic (A = -0.75) in float
__host__ __device__ inline void cubic_coeffs(float x, float *k) {
    const float A = -0.75f, x1 = fadd(x, 1.f), y = fsub(1.f, x);
    k[0] = fsub(fmul(fadd(fmul(fsub(fmul(A, x1), 5.f * A), x1), 8.f * A), x1), 4.f * A);
    k[1] = fadd(fmul(fmul(fsub(fmul(A + 2.f, x), A + 3.f), x), x), 1.f);
    k[2] = fadd(fmul(fmul(fsub(fmul(A + 2.f, y), A + 3.f), y), y), 1.f);
    k[3] = fsub(fsub(fsub(1.f, k[0]), k[1]), k[2]);
}

struct CubicAxis { int i[4]; float k[4]; };

// cv2.resize INTER_CUBIC's taps of destination index d (src samples -> dst samples): the four sources around
// floor((d + 0.5) * src / dst - 0.5), clamped to the edge; the fraction is kept at the borders
__host__ __device__ inline CubicAxis cubic_axis(int d, int dst, int src) {
    const double scale = 1.0 / ((double)dst / (double)src);
    float f = (float)mr_input::src_coord(d, scale);
    const int s = (int)floorf(f);
    f = fsub(f, (float)s);
    CubicAxis a;
    for (int j = 0; j < 4; ++j) a.i[j] = iclamp(s - 1 + j, 0, src - 1);
    cubic_coeffs(f, a.k);
    return a;
}

// cv2.resize(img, (dw, dh), INTER_CUBIC) at (r, c), three channels: each source row's horizontal sum, left to right, then the
// vertical one from the last row up, as cv2's vectorised VResizeCubicVec_32f adds them (its scalar tail, the last
// width * 3 % lanes values of a row, adds from the first row down; DESIGN §7)
template <typename S>
__host__ __device__ inline void cubic_pixel(const S *img, int w, const CubicAxis &ay, const CubicAxis &ax, float *out) {
    for (int ch = 0; ch < 3; ++ch) {
        float row[4];
        for (int j = 0; j < 4; ++j) {
            const int y = ay.i[j];
            row[j] = fadd(fadd(fadd(fmul(px(img, w, y, ax.i[0], ch), ax.k[0]), fmul(px(img, w, y, ax.i[1], ch), ax.k[1])),
                               fmul(px(img, w, y, ax.i[2], ch), ax.k[2])),
                          fmul(px(img, w, y, ax.i[3], ch), ax.k[3]));
        }
        out[ch] = fadd(fmul(row[0], ay.k[0]), fadd(fmul(row[1], ay.k[1]), fadd(fmul(row[2], ay.k[2]), fmul(row[3], ay.k[3]))));
    }
}

// cv2.resize INTER_LINEAR's value from its four taps (input_core.cuh's axis_taps): the rows first, then the column
__host__ __device__ inline float linear_blend(float t00, float t01, float t10, float t11, const mr_input::Axis &lx,
                                              const mr_input::Axis &ly) {
    const float r0 = fadd(fmul(t00, lx.w0), fmul(t01, lx.w1));
    const float r1 = fadd(fmul(t10, lx.w0), fmul(t11, lx.w1));
    return fadd(fmul(r0, ly.w0), fmul(r1, ly.w1));
}

// The normalised output pixel (y, x) of a [3, out_h, out_w] canvas, three channels (out[c]).
//   training:   src is the warped h x w image; the value is cv2.resize INTER_LINEAR of the crop of its INTER_CUBIC resize
//               to hs x ws, placed at the top left of a zero canvas;
//   validation: src is the input; the value is its INTER_CUBIC resize to out_h x out_w.
template <typename S>
__host__ __device__ inline void output_pixel(const Params &P, const Geom &g, const S *src, int y, int x, float *out) {
    float v[3] = {0.f, 0.f, 0.f};
    if (g.status == 0) {
        if (P.mode != 0) {
            cubic_pixel(src, g.w, cubic_axis(y, g.hs, g.h), cubic_axis(x, g.ws, g.w), v);
        } else if (y < g.oh && x < g.ow) {
            const mr_input::Axis lx = mr_input::axis_taps(x, g.ow, g.cw, true), ly = mr_input::axis_taps(y, g.oh, g.ch, false);
            const CubicAxis cx0 = cubic_axis(g.cx + lx.i0, g.ws, g.w), cx1 = cubic_axis(g.cx + lx.i1, g.ws, g.w);
            const CubicAxis cy0 = cubic_axis(g.cy + ly.i0, g.hs, g.h), cy1 = cubic_axis(g.cy + ly.i1, g.hs, g.h);
            float t00[3], t01[3], t10[3], t11[3];
            cubic_pixel(src, g.w, cy0, cx0, t00);
            cubic_pixel(src, g.w, cy0, cx1, t01);
            cubic_pixel(src, g.w, cy1, cx0, t10);
            cubic_pixel(src, g.w, cy1, cx1, t11);
            for (int c = 0; c < 3; ++c) v[c] = linear_blend(t00[c], t01[c], t10[c], t11[c], lx, ly);
        }
    }
    for (int c = 0; c < 3; ++c) out[c] = mr_input::normalize_value(v[c], P.mean[c]);
}

}  // namespace mr_dbbatch
