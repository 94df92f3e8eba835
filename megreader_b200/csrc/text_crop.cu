// Text crops for recognition on the device: ImageCropper.crop (data/crop_file_dataset.py:85-124) for every quad of a ragged
// batch of images (text_crop_core.cuh holds the arithmetic).
//   1. text_crop_rows_kernel: per image the shape checks and its number of quads, their exclusive prefix sum (the rows of the
//      output, in (image, quad) order), the total and the overflow past the capacity;
//   2. text_crop_setup_kernel: per row the quad's rectangle, perspective matrix, crop size, turn and resize width, and its owner;
//   3. text_crop_sample_kernel: per output pixel the resize of the turned crop, each tap a warpPerspective sample of the
//      source, then the normalisation.  Rows past the total are not touched.
// Nothing is read back to the host, so the call can be captured in a CUDA graph and replayed with new images and quads.
#include "common.cuh"
#include "text_crop_core.cuh"

using namespace mr;
using mr_textcrop::Crop;

namespace {

constexpr int kThreads = 256;
constexpr int kMaxRows = 65535;          // the sample grid's y extent

int64_t r256(int64_t b) { return round_up(b, 256); }

struct Layout {
    int64_t o_rows, o_crop, total;
};

Layout layout(int64_t N, int64_t cap) {
    Layout l;
    int64_t o = 0;
    l.o_rows = o; o += r256((N + 1) * 4);
    l.o_crop = o; o += r256(cap * (int64_t)sizeof(Crop));
    l.total = o;
    return l;
}

// One thread: every image's status and quad count, their prefix sum into rows[N + 1], the total.  K > 0: quads [N, K, 4, 2]
// with count[n] quads of image n; K == 0: quads [quad_rows, 4, 2] with image n's at count[n] .. count[n + 1] (offsets).
__global__ void text_crop_rows_kernel(int N, const int *__restrict__ shapes, const int64_t *__restrict__ img_off, int64_t img_elems,
                                      const int *__restrict__ count, int K, int64_t quad_rows, int cap, int *rows, int *total,
                                      int *status) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    int run = 0;
    for (int n = 0; n < N; ++n) {
        const int h = shapes[2 * n], w = shapes[2 * n + 1];
        int st = 0, k;
        if (K > 0) {
            k = count[n];
            if (k < 0 || k > K) st |= mr_textcrop::kBadCount;
        } else {
            const int lo = count[n], hi = count[n + 1];
            k = hi - lo;
            if (lo < 0 || hi < lo || hi > quad_rows) st |= mr_textcrop::kBadCount;
        }
        if (h < 1 || w < 1 || h > mr_textcrop::kMaxSide || w > mr_textcrop::kMaxSide) st |= mr_textcrop::kBadShape;
        else if (img_off[n] < 0 || img_off[n] + (int64_t)h * w * 3 > img_elems) st |= mr_textcrop::kBadPixels;
        if (st) k = 0;
        rows[n] = run;
        if (run + k > cap) st |= mr_textcrop::kOverflow;
        run += k;
        status[n] = st;
    }
    rows[N] = run;
    *total = run;
}

// thread r: output row r < min(total, capacity): its image (the last n with rows[n] <= r), quad and crop parameters
template <class Q>
__global__ void __launch_bounds__(kThreads) text_crop_setup_kernel(int N, const int *__restrict__ shapes, const Q *__restrict__ quads,
                                                                   const int *__restrict__ count, int K, const int *__restrict__ rows,
                                                                   int cap, int mode, int out_h, int out_w, Crop *crops, int *owner,
                                                                   int *status) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= cap) return;
    if (r >= rows[N]) {
        owner[2 * r] = owner[2 * r + 1] = -1;
        return;
    }
    int lo = 0, hi = N - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (rows[mid] <= r) lo = mid; else hi = mid - 1;
    }
    const int n = lo, b = r - rows[n];
    const int64_t qi = K > 0 ? (int64_t)n * K + b : (int64_t)count[n] + b;
    float q[8];
    for (int k = 0; k < 8; ++k) q[k] = (float)quads[8 * qi + k];
    Crop c;
    mr_textcrop::setup(q, shapes[2 * n], shapes[2 * n + 1], mode, out_h, out_w, c);
    crops[r] = c;
    owner[2 * r] = n;
    owner[2 * r + 1] = b;
    if (c.flags) atomicOr(status + n, c.flags);
}

// block (x, row): output pixels of one row, all three channels per thread
template <class S>
__global__ void __launch_bounds__(kThreads) text_crop_sample_kernel(const S *__restrict__ images, const int64_t *__restrict__ img_off,
                                                                    const int *__restrict__ shapes, const Crop *__restrict__ crops,
                                                                    const int *__restrict__ owner, const int *__restrict__ total,
                                                                    int out_h, int out_w, double m0, double m1, double m2, float *out) {
    const int r = blockIdx.y;
    if (r >= *total) return;
    __shared__ Crop c;
    if (threadIdx.x == 0) c = crops[r];
    __syncthreads();
    const int n = owner[2 * r];
    const int h = shapes[2 * n], w = shapes[2 * n + 1];
    const S *img = images + img_off[n];
    const double mean[3] = {m0, m1, m2};
    const int64_t plane = (int64_t)out_h * out_w;
    float *o = out + (int64_t)r * 3 * plane;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < plane; i += (int64_t)gridDim.x * blockDim.x) {
        float v[3];
        mr_textcrop::output_pixel(c, img, h, w, out_h, mean, (int)(i / out_w), (int)(i % out_w), v);
        o[i] = v[0];
        o[plane + i] = v[1];
        o[2 * plane + i] = v[2];
    }
}

bool bad_sizes(int64_t N, int64_t cap) { return N < 1 || N > 65535 || cap < 0 || cap > kMaxRows; }

}  // namespace

extern "C" {

int64_t mr_text_crop_workspace_bytes(int64_t N, int64_t capacity) {
    if (bad_sizes(N, capacity)) return 0;
    return layout(N, capacity).total;
}

int mr_text_crop(const void *images, int image_dtype, int64_t image_elems, const int64_t *image_offsets, const int *shapes, int N,
                 const void *quads, int quad_dtype, int64_t quad_rows, int K, const int *count, int capacity, int mode, int out_h,
                 int out_w, double mean0, double mean1, double mean2, void *workspace, int64_t workspace_bytes, float *image_out,
                 int *owner, int *total, int *status, void *stream) {
    if (bad_sizes(N, capacity) || (image_dtype != 0 && image_dtype != 1) || (quad_dtype != 0 && quad_dtype != 1) || (mode != 0 && mode != 1) ||
        out_h < 1 || out_w < 1 || (int64_t)out_h * out_w > ((int64_t)1 << 26) || image_elems < 0 || K < 0 || quad_rows < 0 ||
        (K > 0 && quad_rows != (int64_t)N * K))
        return MR_ERR_BAD_SHAPE;
    const Layout l = layout(N, capacity);
    if (workspace_bytes < l.total) return MR_ERR_BAD_SHAPE;
    if (!images || !image_offsets || !shapes || !count || !workspace || !total || !status) return MR_ERR_NULL_POINTER;
    if (capacity > 0 && (!quads || !image_out || !owner)) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    int *rows = (int *)(ws + l.o_rows);
    Crop *crops = (Crop *)(ws + l.o_crop);
    int rc;
    text_crop_rows_kernel<<<1, 32, 0, st>>>(N, shapes, image_offsets, image_elems, count, K, quad_rows, capacity, rows, total, status);
    if ((rc = check_launch("text_crop rows"))) return rc;
    if (capacity == 0) return MR_OK;
    const int setup_blocks = (int)ceil_div(capacity, kThreads);
    if (quad_dtype == 0)
        text_crop_setup_kernel<int><<<setup_blocks, kThreads, 0, st>>>(N, shapes, (const int *)quads, count, K, rows, capacity, mode, out_h,
                                                                      out_w, crops, owner, status);
    else
        text_crop_setup_kernel<float><<<setup_blocks, kThreads, 0, st>>>(N, shapes, (const float *)quads, count, K, rows, capacity, mode,
                                                                        out_h, out_w, crops, owner, status);
    if ((rc = check_launch("text_crop setup"))) return rc;
    const dim3 grid((unsigned)std::min<int64_t>(ceil_div((int64_t)out_h * out_w, kThreads), 256), capacity);
    if (image_dtype == 0)
        text_crop_sample_kernel<unsigned char><<<grid, kThreads, 0, st>>>((const unsigned char *)images, image_offsets, shapes, crops, owner,
                                                                          total, out_h, out_w, mean0, mean1, mean2, image_out);
    else
        text_crop_sample_kernel<float><<<grid, kThreads, 0, st>>>((const float *)images, image_offsets, shapes, crops, owner, total, out_h,
                                                                  out_w, mean0, mean1, mean2, image_out);
    return check_launch("text_crop sample");
}

}  // extern "C"
