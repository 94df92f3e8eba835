// The DB detector's input batch on the device: seg_detector_db.yaml's AugmentDetectionData, RandomCropData, MakeICDARData
// and NormalizeImage for a ragged batch of decoded images (db_batch_core.cuh holds the arithmetic).
//   1. db_batch_geometry_kernel: one block per image: the shape checks, the augmentation from the draws, the quads through the
//      flip, rotation and resize; in training crop_area's w_array / h_array, their zero indices, the tries, the canvas scale;
//      then the quads on the canvas and which of them the crop keeps, ranked in input order;
//   2. db_batch_offsets_kernel: the kept counts -> the new offsets;
//   3. db_batch_polys_kernel: the kept quads and tags compacted to the new offsets as float64 (MakeICDARData), zero rows after;
//   4. db_batch_warp_kernel (training): the flipped and rotated image, at most the input's size;
//   5. db_batch_sample_kernel: per output pixel the cubic resize, the crop's linear resize (training) and the normalisation.
// Nothing is read back to the host, so the call can be captured in a CUDA graph and replayed with new images and draws.
#include "common.cuh"
#include "db_batch_core.cuh"

using namespace mr;
using mr_dbbatch::Geom;
using mr_dbbatch::Params;

namespace {

constexpr int kThreads = 256;

int64_t r256(int64_t b) { return round_up(b, 256); }

struct Layout {
    int64_t axis_w, axis_h;              // per-image length of the w and h axes: the resized sides' bound
    int64_t o_geom, o_tpoly, o_rank, o_count, o_mark, o_axis, o_warp, total;      // o_count: N counts, then the offsets flag
};

Layout layout(int64_t N, int64_t max_h, int64_t max_w, int64_t cap) {
    Layout l;
    l.axis_w = (int64_t)ceil(mr_dbbatch::kMaxScale * (double)max_w) + 1;
    l.axis_h = (int64_t)ceil(mr_dbbatch::kMaxScale * (double)max_h) + 1;
    int64_t o = 0;
    l.o_geom = o;  o += r256(N * (int64_t)sizeof(Geom));
    l.o_tpoly = o; o += r256(cap * 8 * (int64_t)sizeof(double));
    l.o_rank = o;  o += r256(cap * 4);
    l.o_count = o; o += r256((N + 1) * 4);
    l.o_mark = o;  o += r256(N * (l.axis_w + l.axis_h));
    l.o_axis = o;  o += r256(N * (l.axis_w + l.axis_h) * 4);
    l.o_warp = o;  o += r256(N * max_h * max_w * 3 * 4);
    l.total = o;
    return l;
}

struct Work {
    Geom *geom;
    double *tpoly;
    int *rank, *count;
    unsigned char *mark;
    int *axis;
    float *warp;
    int64_t axis_w, axis_h;
};

Work work(const Layout &l, char *ws) {
    return Work{(Geom *)(ws + l.o_geom), (double *)(ws + l.o_tpoly), (int *)(ws + l.o_rank), (int *)(ws + l.o_count),
                (unsigned char *)(ws + l.o_mark), (int *)(ws + l.o_axis), (float *)(ws + l.o_warp), l.axis_w, l.axis_h};
}

// The zero indices of mark[0..L) in order into axis; returns their count (all threads)
__device__ int zero_indices(const unsigned char *mark, int L, int *axis, int *s_cnt) {
    const int chunk = (L + kThreads - 1) / kThreads, a = min(L, (int)threadIdx.x * chunk), b = min(L, a + chunk);
    int c = 0;
    for (int i = a; i < b; ++i) c += mark[i] == 0;
    s_cnt[threadIdx.x] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int t = 0; t < kThreads; ++t) { const int v = s_cnt[t]; s_cnt[t] = run; run += v; }
        s_cnt[kThreads] = run;
    }
    __syncthreads();
    int o = s_cnt[threadIdx.x];
    for (int i = a; i < b; ++i)
        if (mark[i] == 0) axis[o++] = i;
    const int total = s_cnt[kThreads];
    __syncthreads();
    return total;
}

template <class T>
__global__ void __launch_bounds__(kThreads) db_batch_geometry_kernel(Params P, const int *__restrict__ shapes,
                                                                     const int64_t *__restrict__ img_off, int64_t img_elems,
                                                                     int max_h, int max_w, const T *__restrict__ polys,
                                                                     const unsigned char *__restrict__ tags,
                                                                     const int *__restrict__ offsets, int cap,
                                                                     const float *__restrict__ draws, int n_draws, Work W,
                                                                     int *shape_out, int *crop_out, double *scale_out, int *status) {
    const int n = blockIdx.x;
    __shared__ Geom g;
    __shared__ int s_lo, s_hi;
    __shared__ int s_cnt[kThreads + 1];
    const float *u = draws + (int64_t)n * n_draws;
    if (threadIdx.x == 0) {
        const int h = shapes[2 * n], w = shapes[2 * n + 1];
        int st = 0;
        if (h < 1 || w < 1 || h > max_h || w > max_w) st |= mr_dbbatch::kBadShape;
        else if (img_off[n] < 0 || img_off[n] + (int64_t)h * w * 3 > img_elems) st |= mr_dbbatch::kBadPixels;
        int lo = offsets[n], hi = offsets[n + 1];
        if (!W.count[gridDim.x]) { st |= mr_dbbatch::kBadOffsets; lo = hi = 0; }
        mr_dbbatch::augment_geometry(P, u, st ? 1 : h, st ? 1 : w, g);
        if (g.ws > W.axis_w || g.hs > W.axis_h) st |= mr_dbbatch::kBadShape;
        g.status = st;
        s_lo = lo; s_hi = hi;
    }
    __syncthreads();
    const int lo = s_lo, hi = s_hi;
    double *tp = W.tpoly;
    for (int p = lo + threadIdx.x; p < hi; p += kThreads)
        for (int k = 0; k < 4; ++k)
            mr_dbbatch::augment_point(g, (double)polys[8 * (int64_t)p + 2 * k], (double)polys[8 * (int64_t)p + 2 * k + 1],
                                      tp[8 * (int64_t)p + 2 * k], tp[8 * (int64_t)p + 2 * k + 1]);
    __syncthreads();
    if (P.mode == 0 && g.status == 0) {
        unsigned char *mw = W.mark + (int64_t)n * (W.axis_w + W.axis_h), *mh = mw + W.axis_w;
        int *aw = W.axis + (int64_t)n * (W.axis_w + W.axis_h), *ah = aw + W.axis_w;
        for (int i = threadIdx.x; i < g.ws; i += kThreads) mw[i] = 0;
        for (int i = threadIdx.x; i < g.hs; i += kThreads) mh[i] = 0;
        __syncthreads();
        for (int p = lo; p < hi; ++p) {
            if (tags[p]) continue;
            int x0, x1, y0, y1;
            mr_dbbatch::marked_slices(tp + 8 * (int64_t)p, g.ws, g.hs, x0, x1, y0, y1);
            for (int i = x0 + threadIdx.x; i < x1; i += kThreads) mw[i] = 1;
            for (int i = y0 + threadIdx.x; i < y1; i += kThreads) mh[i] = 1;
        }
        __syncthreads();
        const int nw = zero_indices(mw, g.ws, aw, s_cnt);
        const int nh = zero_indices(mh, g.hs, ah, s_cnt);
        if (threadIdx.x == 0)
            mr_dbbatch::choose_crop(P, u, aw, nw, ah, nh, tp + 8 * (int64_t)lo, tags + lo, hi - lo, g);
    }
    __syncthreads();
    for (int p = lo + threadIdx.x; p < hi; p += kThreads) {
        double *q = tp + 8 * (int64_t)p;
        bool keep = g.status == 0;
        if (keep && P.mode == 0) {
            for (int k = 0; k < 4; ++k) {
                q[2 * k] = mr_dbbatch::crop_coord(q[2 * k], g.cx, g.scale);
                q[2 * k + 1] = mr_dbbatch::crop_coord(q[2 * k + 1], g.cy, g.scale);
            }
            keep = !mr_dbbatch::poly_outside_rect(q, 0., 0., (double)g.ow, (double)g.oh);
        }
        W.rank[p] = keep ? 0 : -1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int r = 0;
        for (int p = lo; p < hi; ++p)
            if (W.rank[p] >= 0) W.rank[p] = r++;
        W.count[n] = r;
        W.geom[n] = g;
        shape_out[2 * n] = g.status ? shapes[2 * n] : g.h;
        shape_out[2 * n + 1] = g.status ? shapes[2 * n + 1] : g.w;
        crop_out[4 * n] = g.cx; crop_out[4 * n + 1] = g.cy; crop_out[4 * n + 2] = g.cw; crop_out[4 * n + 3] = g.ch;
        scale_out[n] = g.scale;
        status[n] = g.status;
    }
}

// ok = offsets non-decreasing from >= 0 to <= capacity; every image's quads are refused otherwise, so that no slot belongs to
// two images
__global__ void db_batch_check_offsets_kernel(int N, int cap, const int *__restrict__ offsets, int *ok) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        bool good = offsets[0] >= 0 && offsets[N] <= cap;
        for (int n = 0; n < N; ++n) good = good && offsets[n] <= offsets[n + 1];
        *ok = good;
    }
}

__global__ void db_batch_offsets_kernel(int N, const int *__restrict__ count, int *offsets_out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        int run = 0;
        offsets_out[0] = 0;
        for (int n = 0; n < N; ++n) { run += count[n]; offsets_out[n + 1] = run; }
    }
}

// thread i: input slot i (its kept quad to its new row) and output row i (zero when past the new total)
__global__ void db_batch_polys_kernel(int N, int cap, const int *__restrict__ offsets, const Geom *__restrict__ geom,
                                      const int *__restrict__ rank, const double *__restrict__ tpoly,
                                      const unsigned char *__restrict__ tags, const int *__restrict__ offsets_out,
                                      double *polys_out, unsigned char *tags_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    const int total = offsets_out[N];
    if (i >= total) {
        for (int k = 0; k < 8; ++k) polys_out[8 * (int64_t)i + k] = 0.;
        tags_out[i] = 0;
    }
    // the image of slot i: the last n with offsets[n] <= i, provided the offsets were accepted
    int lo = 0, hi = N - 1;
    if (geom[0].status & mr_dbbatch::kBadOffsets || i < offsets[0]) return;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (offsets[mid] <= i) lo = mid; else hi = mid - 1;
    }
    if (i >= offsets[lo + 1] || rank[i] < 0) return;
    const int64_t row = offsets_out[lo] + rank[i];
    for (int k = 0; k < 8; ++k) polys_out[8 * row + k] = tpoly[8 * (int64_t)i + k];
    tags_out[row] = tags[i];
}

template <class S>
__global__ void db_batch_warp_kernel(const S *__restrict__ images, const int64_t *__restrict__ img_off, const Geom *__restrict__ geom,
                                     int64_t stride, float *warp) {
    const int n = blockIdx.y;
    const Geom &g = geom[n];
    if (g.status) return;
    const S *img = images + img_off[n];
    float *out = warp + (int64_t)n * stride;
    const int64_t total = (int64_t)g.h * g.w;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / g.w), x = (int)(i % g.w);
        mr_dbbatch::warp_pixel(img, g.h, g.w, g.flip != 0, g.A, y, x, out + 3 * i);
    }
}

template <class S>
__global__ void db_batch_sample_kernel(Params P, const S *__restrict__ src, const int64_t *__restrict__ src_off, int64_t stride,
                                       const Geom *__restrict__ geom, float *out) {
    const int n = blockIdx.y;
    const Geom g = geom[n];
    const int64_t plane = (int64_t)P.out_h * P.out_w;
    const S *img = src + (src_off ? (g.status ? 0 : src_off[n]) : (int64_t)n * stride);
    float *o = out + (int64_t)n * 3 * plane;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < plane; i += (int64_t)gridDim.x * blockDim.x) {
        float v[3];
        mr_dbbatch::output_pixel(P, g, img, (int)(i / P.out_w), (int)(i % P.out_w), v);
        o[i] = v[0];
        o[plane + i] = v[1];
        o[2 * plane + i] = v[2];
    }
}

bool bad_sizes(int64_t N, int64_t max_h, int64_t max_w, int64_t cap) {
    return N <= 0 || N > 65535 || max_h <= 0 || max_w <= 0 || max_h > 16384 || max_w > 16384 || cap < 0 || cap > ((int64_t)1 << 24) ||
           N * max_h * max_w > ((int64_t)1 << 34);
}

}  // namespace

extern "C" {

int64_t mr_db_batch_workspace_bytes(int64_t N, int64_t max_h, int64_t max_w, int64_t capacity) {
    if (bad_sizes(N, max_h, max_w, capacity)) return 0;
    return layout(N, max_h, max_w, capacity).total;
}

int mr_db_batch(const void *images, int image_dtype, int64_t image_elems, const int64_t *image_offsets, const int *shapes, int N,
                int max_h, int max_w, const void *polygons, int poly_dtype, const unsigned char *ignore_tags, const int *offsets,
                int capacity, const float *draws, int n_draws, int mode, int out_h, int out_w, int max_tries,
                double min_crop_side_ratio, double flip_p, double rotate_lo, double rotate_hi, double scale_lo, double scale_hi,
                double mean0, double mean1, double mean2, void *workspace, int64_t workspace_bytes, float *image_out,
                double *polygons_out, unsigned char *ignore_out, int *offsets_out, int *shape_out, int *crop_out, double *scale_out,
                int *status, void *stream) {
    if (bad_sizes(N, max_h, max_w, capacity) || (image_dtype != 0 && image_dtype != 1) || (poly_dtype != 0 && poly_dtype != 1) ||
        (mode != 0 && mode != 1) || out_h < 1 || out_w < 1 || (int64_t)out_h * out_w > ((int64_t)1 << 26) || image_elems < 0)
        return MR_ERR_BAD_SHAPE;
    if (mode == 0 && (max_tries < 1 || max_tries > 1000 || n_draws < mr_dbbatch::draws_needed(max_tries) || !(scale_lo > 0.) ||
                      !(scale_hi >= scale_lo) || scale_hi > mr_dbbatch::kMaxScale || !(rotate_hi >= rotate_lo) || rotate_lo < -180. ||
                      rotate_hi > 180. || !(min_crop_side_ratio >= 0.)))
        return MR_ERR_BAD_SHAPE;
    if (mode == 1 && ((double)out_h > mr_dbbatch::kMaxScale * max_h || (double)out_w > mr_dbbatch::kMaxScale * max_w)) return MR_ERR_BAD_SHAPE;
    if (!images || !image_offsets || !shapes || !offsets || !workspace || !image_out || !offsets_out || !shape_out || !crop_out ||
        !scale_out || !status || (mode == 0 && !draws))
        return MR_ERR_NULL_POINTER;
    if (capacity > 0 && (!polygons || !ignore_tags || !polygons_out || !ignore_out)) return MR_ERR_NULL_POINTER;
    const Layout l = layout(N, max_h, max_w, capacity);
    if (workspace_bytes < l.total) return MR_ERR_BAD_SHAPE;
    Params P;
    P.mode = mode; P.out_h = out_h; P.out_w = out_w; P.max_tries = max_tries; P.min_ratio = min_crop_side_ratio;
    P.flip_p = flip_p; P.rot_lo = rotate_lo; P.rot_hi = rotate_hi; P.scale_lo = scale_lo; P.scale_hi = scale_hi;
    P.mean[0] = mean0; P.mean[1] = mean1; P.mean[2] = mean2;
    const Work W = work(l, (char *)workspace);
    cudaStream_t st = (cudaStream_t)stream;
    const int nd = mode == 0 ? n_draws : 0;
    int rc;
    db_batch_check_offsets_kernel<<<1, 32, 0, st>>>(N, capacity, offsets, W.count + N);
    if ((rc = check_launch("db_batch check"))) return rc;
    if (poly_dtype == 0)
        db_batch_geometry_kernel<float><<<N, kThreads, 0, st>>>(P, shapes, image_offsets, image_elems, max_h, max_w, (const float *)polygons,
                                                              ignore_tags, offsets, capacity, draws, nd, W, shape_out, crop_out, scale_out, status);
    else
        db_batch_geometry_kernel<double><<<N, kThreads, 0, st>>>(P, shapes, image_offsets, image_elems, max_h, max_w, (const double *)polygons,
                                                               ignore_tags, offsets, capacity, draws, nd, W, shape_out, crop_out, scale_out, status);
    if ((rc = check_launch("db_batch geometry"))) return rc;
    db_batch_offsets_kernel<<<1, 32, 0, st>>>(N, W.count, offsets_out);
    if ((rc = check_launch("db_batch offsets"))) return rc;
    if (capacity > 0) {
        db_batch_polys_kernel<<<(int)ceil_div(capacity, kThreads), kThreads, 0, st>>>(N, capacity, offsets, W.geom, W.rank, W.tpoly,
                                                                                     ignore_tags, offsets_out, polygons_out, ignore_out);
        if ((rc = check_launch("db_batch polygons"))) return rc;
    }
    const int64_t stride = (int64_t)max_h * max_w * 3;
    const dim3 sample_grid((unsigned)std::min<int64_t>(ceil_div((int64_t)out_h * out_w, kThreads), 1024), N);
    if (mode == 0) {
        const dim3 warp_grid((unsigned)std::min<int64_t>(ceil_div((int64_t)max_h * max_w, kThreads), 2048), N);
        if (image_dtype == 0)
            db_batch_warp_kernel<unsigned char><<<warp_grid, kThreads, 0, st>>>((const unsigned char *)images, image_offsets, W.geom, stride, W.warp);
        else
            db_batch_warp_kernel<float><<<warp_grid, kThreads, 0, st>>>((const float *)images, image_offsets, W.geom, stride, W.warp);
        if ((rc = check_launch("db_batch warp"))) return rc;
        db_batch_sample_kernel<float><<<sample_grid, kThreads, 0, st>>>(P, W.warp, nullptr, stride, W.geom, image_out);
    } else if (image_dtype == 0) {
        db_batch_sample_kernel<unsigned char><<<sample_grid, kThreads, 0, st>>>(P, (const unsigned char *)images, image_offsets, 0, W.geom,
                                                                                image_out);
    } else {
        db_batch_sample_kernel<float><<<sample_grid, kThreads, 0, st>>>(P, (const float *)images, image_offsets, 0, W.geom, image_out);
    }
    return check_launch("db_batch sample");
}

}  // extern "C"
