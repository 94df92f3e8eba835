// Host-side harness: runs the PRODUCT's per-quad and per-pixel routines of the text crop (megreader_b200/csrc/text_crop_core.cuh,
// the code the CUDA kernels in text_crop.cu execute) on the CPU, so that tests can compare them with cv2 and the oracle without
// a GPU.  Built on demand with g++ -ffp-contract=off.
#include "text_crop_core.cuh"

using namespace mr_textcrop;

static const double kMean[3] = {122.67891434, 116.66876762, 104.00698793};

extern "C" {

// The setup of k quads (float32 [k, 4, 2]) for an img_h x img_w source: box [k, 8], sides [k, 2] (float32 w, h), size [k, 4]
// (crop w, h, resize input h, w), ints [k, 3] (turned, valid_w, flags), P and M [k, 9]
void host_setup(const float *q, int k, int img_h, int img_w, int mode, int out_h, int out_w, float *box, float *sides, int *size,
                int *ints, double *P, double *M) {
    for (int i = 0; i < k; ++i) {
        Crop c;
        setup(q + 8 * i, img_h, img_w, mode, out_h, out_w, c);
        for (int j = 0; j < 8; ++j) box[8 * i + j] = c.box[j];
        sides[2 * i] = c.w; sides[2 * i + 1] = c.h;
        size[4 * i] = c.cw; size[4 * i + 1] = c.ch; size[4 * i + 2] = c.rh; size[4 * i + 3] = c.rw;
        ints[3 * i] = c.turned; ints[3 * i + 1] = c.valid_w; ints[3 * i + 2] = c.flags;
        for (int j = 0; j < 9; ++j) { P[9 * i + j] = c.P[j]; M[9 * i + j] = c.M[j]; }
    }
}

// cv2.warpPerspective(img, P, (dw, dh)) of an h x w x 3 image (dtype 0 uint8, 1 float32) as float32 [dh, dw, 3]
void host_warp(const void *img, int dtype, int h, int w, const double *P, int dw, int dh, float *out) {
    Crop c;
    invert3(P, c.M);
    c.cw = dw; c.ch = dh;
    c.bw = warp_block_width(dw, dh);
    for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x) {
            float *o = out + ((int64_t)y * dw + x) * 3;
            if (dtype == 0) warp_sample((const unsigned char *)img, h, w, c, x, y, o);
            else warp_sample((const float *)img, h, w, c, x, y, o);
        }
}

// ImageCropper.crop(img, quad) as the kernels compute it: float32 [out_h, out_w, 3] (HWC, as the reference returns it)
void host_crop(const void *img, int dtype, int h, int w, const float *quad, int mode, int out_h, int out_w, float *out) {
    Crop c;
    setup(quad, h, w, mode, out_h, out_w, c);
    for (int y = 0; y < out_h; ++y)
        for (int x = 0; x < out_w; ++x) {
            float *o = out + ((int64_t)y * out_w + x) * 3;
            if (dtype == 0) output_pixel(c, (const unsigned char *)img, h, w, out_h, kMean, y, x, o);
            else output_pixel(c, (const float *)img, h, w, out_h, kMean, y, x, o);
        }
}

}  // extern "C"
