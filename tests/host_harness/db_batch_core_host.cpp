// Host-side harness: runs the PRODUCT's per-image and per-pixel routines of the DB input batch
// (megreader_b200/csrc/db_batch_core.cuh, the code the CUDA kernels in db_batch.cu execute) on the CPU, so that tests can
// compare them with cv2, numpy and the oracle without a GPU.  Built on demand with g++ -ffp-contract=off.
#include <vector>

#include "db_batch_core.cuh"

using namespace mr_dbbatch;

static Params params(int mode, int out_h, int out_w, int max_tries, double min_ratio, double flip_p, double rot_lo, double rot_hi,
                     double scale_lo, double scale_hi) {
    Params P;
    P.mode = mode; P.out_h = out_h; P.out_w = out_w; P.max_tries = max_tries; P.min_ratio = min_ratio;
    P.flip_p = flip_p; P.rot_lo = rot_lo; P.rot_hi = rot_hi; P.scale_lo = scale_lo; P.scale_hi = scale_hi;
    P.mean[0] = 122.67891434; P.mean[1] = 116.66876762; P.mean[2] = 104.00698793;
    return P;
}

extern "C" {

// The geometry of one h x w image as the geometry kernel computes it: polys [k, 4, 2] float64 with tags [k]; writes
// ints[9] = (hs, ws, flip, cx, cy, cw, ch, oh, ow), *scale, aug [k, 4, 2] (after the augmentation), out [k, 4, 2] (on the
// canvas) and keep [k]
void host_geometry(int mode, int out_h, int out_w, int max_tries, double min_ratio, double flip_p, double rot_lo, double rot_hi,
                   double scale_lo, double scale_hi, const float *u, int h, int w, const double *polys, const unsigned char *tags, int k,
                   int *ints, double *scale, double *aug, double *out, unsigned char *keep) {
    const Params P = params(mode, out_h, out_w, max_tries, min_ratio, flip_p, rot_lo, rot_hi, scale_lo, scale_hi);
    Geom g;
    augment_geometry(P, u, h, w, g);
    for (int p = 0; p < k; ++p)
        for (int j = 0; j < 4; ++j) augment_point(g, polys[8 * p + 2 * j], polys[8 * p + 2 * j + 1], aug[8 * p + 2 * j], aug[8 * p + 2 * j + 1]);
    if (mode == 0) {
        std::vector<unsigned char> mw(g.ws, 0), mh(g.hs, 0);
        for (int p = 0; p < k; ++p) {
            if (tags[p]) continue;
            int x0, x1, y0, y1;
            marked_slices(aug + 8 * p, g.ws, g.hs, x0, x1, y0, y1);
            for (int i = x0; i < x1; ++i) mw[i] = 1;
            for (int i = y0; i < y1; ++i) mh[i] = 1;
        }
        std::vector<int> aw, ah;
        for (int i = 0; i < g.ws; ++i) if (!mw[i]) aw.push_back(i);
        for (int i = 0; i < g.hs; ++i) if (!mh[i]) ah.push_back(i);
        choose_crop(P, u, aw.data(), (int)aw.size(), ah.data(), (int)ah.size(), aug, tags, k, g);
    }
    for (int p = 0; p < k; ++p) {
        double *q = out + 8 * p;
        for (int j = 0; j < 8; ++j) q[j] = aug[8 * p + j];
        keep[p] = 1;
        if (mode == 0) {
            for (int j = 0; j < 4; ++j) {
                q[2 * j] = crop_coord(q[2 * j], g.cx, g.scale);
                q[2 * j + 1] = crop_coord(q[2 * j + 1], g.cy, g.scale);
            }
            keep[p] = !poly_outside_rect(q, 0., 0., (double)g.ow, (double)g.oh);
        }
    }
    const int v[9] = {g.hs, g.ws, g.flip, g.cx, g.cy, g.cw, g.ch, g.oh, g.ow};
    for (int i = 0; i < 9; ++i) ints[i] = v[i];
    *scale = g.scale;
}

// cv2.warpAffine(flip(img) if flip else img, rotation matrix of deg, (w, h)) on a float32 h x w x 3 image
void host_warp(const float *img, int h, int w, int flip, double deg, float *out) {
    double M[6], A[6];
    rotation_matrix(deg, w, h, M);
    invert_affine(M, A);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) warp_pixel(img, h, w, flip != 0, A, y, x, out + ((int64_t)y * w + x) * 3);
}

// The forward matrix of imgaug's rotation, for the oracle
void host_rotation_matrix(double deg, int w, int h, double *M) { rotation_matrix(deg, w, h, M); }

// cv2.resize(img, (dw, dh), interpolation=INTER_CUBIC) on a float32 h x w x 3 image
void host_cubic(const float *img, int h, int w, int dh, int dw, float *out) {
    for (int y = 0; y < dh; ++y) {
        const CubicAxis ay = cubic_axis(y, dh, h);
        for (int x = 0; x < dw; ++x) cubic_pixel(img, w, ay, cubic_axis(x, dw, w), out + ((int64_t)y * dw + x) * 3);
    }
}

// cv2.resize(img, (dw, dh)) (INTER_LINEAR) on a float32 h x w x 3 image
void host_linear(const float *img, int h, int w, int dh, int dw, float *out) {
    for (int y = 0; y < dh; ++y) {
        const mr_input::Axis ly = mr_input::axis_taps(y, dh, h, false);
        for (int x = 0; x < dw; ++x) {
            const mr_input::Axis lx = mr_input::axis_taps(x, dw, w, true);
            for (int c = 0; c < 3; ++c)
                out[((int64_t)y * dw + x) * 3 + c] = linear_blend(px(img, w, ly.i0, lx.i0, c), px(img, w, ly.i0, lx.i1, c),
                                                                  px(img, w, ly.i1, lx.i0, c), px(img, w, ly.i1, lx.i1, c), lx, ly);
        }
    }
}

// The normalised [3, out_h, out_w] output of one image as the warp and sample kernels compute it, from a float32 h x w x 3
// input and the geometry host_geometry returned (ints, scale) and the draws' flip and angle
void host_output(int mode, int out_h, int out_w, double rot_lo, double rot_hi, const float *u, const float *img, int h, int w,
                 const int *ints, double scale, float *out) {
    Params P = params(mode, out_h, out_w, 1, 0., 0., rot_lo, rot_hi, 1., 1.);
    Geom g;
    augment_geometry(P, u, h, w, g);
    g.hs = ints[0]; g.ws = ints[1]; g.flip = ints[2]; g.cx = ints[3]; g.cy = ints[4]; g.cw = ints[5]; g.ch = ints[6];
    g.oh = ints[7]; g.ow = ints[8]; g.scale = scale;
    std::vector<float> warped;
    const float *src = img;
    if (mode == 0) {
        warped.resize((size_t)h * w * 3);
        for (int y = 0; y < h; ++y)
            for (int x = 0; x < w; ++x) warp_pixel(img, h, w, g.flip != 0, g.A, y, x, warped.data() + ((int64_t)y * w + x) * 3);
        src = warped.data();
    }
    const int64_t plane = (int64_t)out_h * out_w;
    for (int y = 0; y < out_h; ++y)
        for (int x = 0; x < out_w; ++x) {
            float v[3];
            output_pixel(P, g, src, y, x, v);
            for (int c = 0; c < 3; ++c) out[c * plane + (int64_t)y * out_w + x] = v[c];
        }
}

}  // extern "C"
