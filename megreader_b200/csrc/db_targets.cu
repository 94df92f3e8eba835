// The DB detector's training targets on the device: MakeSegDetectionData (data/processes/make_seg_detection_data.py:21-100)
// and MakeBorderMap (make_border_map.py:24-121) for a whole batch, after RandomCropData.
//   1. db_polygon_kernel: one thread per polygon slot: validate_polygons, the min-side test, the shrink distance, the shrink
//      and the pad with Clipper's clean-up (db_targets_core.cuh), written as vertex lists into the workspace;
//   2. db_maps_init_kernel: gt = 0, mask = 1, thresh_map = 0, thresh_mask = 0;
//   3. db_fill_kernel: one block per (polygon, fill): the ignored quad into mask (0), the shrunk polygon into gt (1), the
//      padded polygon into thresh_mask (1), each as cv2.fillPoly draws it, with every pixel decided independently;
//   4. db_border_kernel: one block per (polygon, band of rows of its padded box clipped to the image): the per-pixel
//      1 - min clip(distance / d, 0, 1), merged into thresh_map with an integer atomicMax on the float bits (every value is
//      >= 0 and np.fmax over polygons is order-free; NaN pixels leave the canvas unchanged, as np.fmax does);
//   5. db_thresh_scale_kernel: thresh_map * (thresh_max - thresh_min) + thresh_min in float32.
// The polygons are packed [capacity, 4, 2] with device offsets [N + 1], so a captured graph replays with new polygons; no
// step reads anything back to the host.
#include "common.cuh"
#include "db_targets_core.cuh"

using namespace mr;

namespace {

constexpr int kBorderBands = 8;         // blocks per polygon of the border map

int64_t r256(int64_t b) { return round_up(b, 256); }

// Per-slot workspace, in 4-byte words: the raw path, the clean-up scratch, the shrunk and padded polygons
struct SlotLayout {
    mr_dbtgt::Caps c;
    int64_t o_rx, o_ry, o_cre, o_crt, o_crx, o_cry, o_s, o_used, o_l, o_sh, o_pad, words;
};

SlotLayout slot_layout(int H, int W) {
    SlotLayout l;
    l.c = mr_dbtgt::caps_for(H > W ? H : W);
    const int64_t R = l.c.raw, C = 2 * (int64_t)l.c.cross, S = l.c.pieces;
    int64_t o = 0;
    l.o_rx = o;   o += R;
    l.o_ry = o;   o += R;
    l.o_cre = o;  o += C;
    o = round_up(o, 2);
    l.o_crt = o;  o += 2 * C;
    l.o_crx = o;  o += C;
    l.o_cry = o;  o += C;
    l.o_s = o;    o += 4 * S;
    l.o_used = o; o += ceil_div(S, 4);
    l.o_l = o;    o += 2 * S;
    l.o_sh = o;   o += 2 * S;
    l.o_pad = o;  o += 2 * S;
    l.words = round_up(o, 2);
    return l;
}

// Per-slot results of db_polygon_kernel
struct SlotInfo {
    int image, n_shrink, n_pad, status;
    int qi[8];                  // the validated quad astype(np.int32), for the mask fill
    int box[4];                 // padded polygon's xmin, ymin, xmax, ymax
    double distance;
};

struct Layout {
    SlotLayout s;
    int64_t o_info, o_edges, o_slots, total;
};

Layout layout(int64_t cap, int H, int W) {
    Layout l;
    l.s = slot_layout(H, W);
    int64_t o = 0;
    l.o_info = o;  o += r256(cap * (int64_t)sizeof(SlotInfo));
    l.o_edges = o; o += r256(3 * cap * (int64_t)l.s.c.pieces * (int64_t)sizeof(mr_dbtgt::PolyEdge));
    l.o_slots = o; o += r256(cap * l.s.words * 4);
    l.total = o;
    return l;
}

template <class T>
__global__ void db_polygon_kernel(const T *__restrict__ polys, const unsigned char *__restrict__ ignore_in,
                                  const int *__restrict__ offsets, int N, int H, int W, int cap, double shrink_k, double min_text,
                                  SlotLayout sl, int *slots, SlotInfo *info, T *polys_out, unsigned char *ignore_out, int *status_out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= cap) return;
    SlotInfo si;
    si.n_shrink = si.n_pad = si.status = 0;
    si.distance = 0.;
    for (int k = 0; k < 8; ++k) si.qi[k] = 0;
    for (int k = 0; k < 4; ++k) si.box[k] = 0;
    // image of the slot: the last n with offsets[n] <= p (offsets clamped to [0, cap]; empty images are skipped)
    auto off = [&](int n) { const int v = offsets[n]; return v < 0 ? 0 : v > cap ? cap : v; };
    si.image = -1;
    if (p < off(N)) {
        int lo = 0, hi = N - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (off(mid) <= p) lo = mid; else hi = mid - 1;
        }
        si.image = lo;
    }
    T q[8];
    for (int k = 0; k < 8; ++k) q[k] = polys[8 * (int64_t)p + k];
    if (si.image >= 0) {
        int *w = slots + (int64_t)p * sl.words;
        mr_dbtgt::CleanScratch s;
        s.cr_e = w + sl.o_cre;
        s.cr_t = (double *)(w + sl.o_crt);
        s.cr_x = w + sl.o_crx;
        s.cr_y = w + sl.o_cry;
        const int S = sl.c.pieces;
        s.sx0 = w + sl.o_s; s.sy0 = s.sx0 + S; s.sx1 = s.sy0 + S; s.sy1 = s.sx1 + S;
        s.used = (unsigned char *)(w + sl.o_used);
        s.lx = w + sl.o_l; s.ly = s.lx + S;
        s.n_cap = sl.c.raw; s.c_cap = sl.c.cross; s.s_cap = S;
        int *sx = w + sl.o_sh, *px = w + sl.o_pad;
        si.status = mr_dbtgt::polygon_targets(q, ignore_in[p] != 0, H, W, shrink_k, min_text, sl.c, w + sl.o_rx, w + sl.o_ry, s,
                                              sx, sx + S, &si.n_shrink, px, px + S, &si.n_pad, &si.distance);
        for (int k = 0; k < 8; ++k) si.qi[k] = (int)q[k];
        if (si.n_pad > 0) {
            int x0 = px[0], x1 = px[0], y0 = px[S], y1 = px[S];
            for (int k = 1; k < si.n_pad; ++k) {
                x0 = min(x0, px[k]); x1 = max(x1, px[k]);
                y0 = min(y0, px[S + k]); y1 = max(y1, px[S + k]);
            }
            si.box[0] = x0; si.box[1] = y0; si.box[2] = x1; si.box[3] = y1;
        }
    }
    info[p] = si;
    for (int k = 0; k < 8; ++k) polys_out[8 * (int64_t)p + k] = q[k];
    ignore_out[p] = si.image >= 0 ? mr_dbtgt::status_ignored(si.status) : ignore_in[p];
    status_out[p] = si.status;
}

__global__ void db_maps_init_kernel(int64_t total, float *gt, float *mask, float *thresh_map, float *thresh_mask) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        gt[i] = 0.f;
        mask[i] = 1.f;
        thresh_map[i] = 0.f;
        thresh_mask[i] = 0.f;
    }
}

// blockIdx.x = slot, blockIdx.y = 0: the ignored quad into mask (0); 1: the shrunk polygon into gt (1); 2: the padded polygon
// into thresh_mask (1)
__global__ void db_fill_kernel(const SlotInfo *__restrict__ info, const int *__restrict__ slots, SlotLayout sl, int H, int W,
                               mr_dbtgt::PolyEdge *edges, float *gt, float *mask, float *thresh_mask) {
    const int p = blockIdx.x, job = blockIdx.y;
    const SlotInfo &si = info[p];
    if (si.image < 0) return;
    const bool ignored = mr_dbtgt::status_ignored(si.status);
    const int S = sl.c.pieces;
    const int *w = slots + (int64_t)p * sl.words;
    int qx[4], qy[4];
    for (int k = 0; k < 4; ++k) { qx[k] = si.qi[2 * k]; qy[k] = si.qi[2 * k + 1]; }
    const int *xs = qx, *ys = qy;
    int n = 4;
    float *img = mask, value = 0.f;
    if (job == 0) {
        if (!ignored) return;
    } else if (job == 1) {
        if (ignored || si.n_shrink == 0) return;
        xs = w + sl.o_sh; ys = xs + S; n = si.n_shrink;
        img = gt; value = 1.f;
    } else {
        if (ignored || si.n_pad == 0) return;
        xs = w + sl.o_pad; ys = xs + S; n = si.n_pad;
        img = thresh_mask; value = 1.f;
    }
    img += (int64_t)si.image * H * W;
    mr_dbtgt::PolyEdge *e = edges + ((int64_t)p * 3 + job) * S;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        e[i] = mr_dbtgt::fill_edge(xs, ys, n, i, W, H, [&](int x, int y) { img[(int64_t)y * W + x] = value; });
    __syncthreads();
    int y_lo, y_hi, x_lo, x_hi;
    if (!mr_dbtgt::fill_bounds(e, n, W, H, y_lo, y_hi, x_lo, x_hi)) return;
    const int64_t bw = x_hi - x_lo + 1, npx = (int64_t)(y_hi - y_lo) * bw;
    for (int64_t i = threadIdx.x; i < npx; i += blockDim.x) {
        const int y = y_lo + (int)(i / bw), x = x_lo + (int)(i % bw);
        if (mr_dbtgt::pixel_filled(e, n, x, y)) img[(int64_t)y * W + x] = value;
    }
}

template <class T>
__global__ void db_border_kernel(const SlotInfo *__restrict__ info, const T *__restrict__ polys, int H, int W, float *canvas) {
    const int p = blockIdx.x;
    const SlotInfo &si = info[p];
    if (si.image < 0 || si.n_pad == 0 || mr_dbtgt::status_ignored(si.status)) return;
    T q[8];
    for (int k = 0; k < 8; ++k) q[k] = polys[8 * (int64_t)p + k];
    const int xmin = si.box[0], ymin = si.box[1], xmax = si.box[2], ymax = si.box[3];
    const int x0 = min(max(0, xmin), W - 1), x1 = min(max(0, xmax), W - 1);
    const int y0 = min(max(0, ymin), H - 1), y1 = min(max(0, ymax), H - 1);
    const int64_t bw = x1 - x0 + 1, rows = y1 - y0 + 1;
    const int64_t r0 = rows * blockIdx.y / gridDim.y, r1 = rows * (blockIdx.y + 1) / gridDim.y;
    unsigned int *c = (unsigned int *)canvas + (int64_t)si.image * H * W;
    for (int64_t i = r0 * bw + threadIdx.x; i < r1 * bw; i += blockDim.x) {
        const int y = y0 + (int)(i / bw), x = x0 + (int)(i % bw);
        const float v = mr_dbtgt::border_value(q, (double)xmin, (double)ymin, (double)(x - xmin), (double)(y - ymin), si.distance);
        if (v == v) atomicMax(c + (int64_t)y * W + x, __float_as_uint(v));
    }
}

__global__ void db_thresh_scale_kernel(int64_t total, float scale, float lo, float *thresh_map) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        thresh_map[i] = __fadd_rn(__fmul_rn(thresh_map[i], scale), lo);
}

constexpr int64_t kMaxPixels = ((int64_t)1 << 28) - 1;

bool bad_sizes(int64_t N, int64_t H, int64_t W, int64_t cap) {
    return N <= 0 || N > 65535 || H <= 0 || W <= 0 || H * W > kMaxPixels || N * H * W > ((int64_t)1 << 40) || cap < 0 ||
           cap > ((int64_t)1 << 24) || H > 65535 || W > 65535;
}

}  // namespace

extern "C" {

int64_t mr_db_targets_workspace_bytes(int64_t N, int64_t H, int64_t W, int64_t capacity) {
    if (bad_sizes(N, H, W, capacity)) return 0;
    const int64_t total = layout(capacity, (int)H, (int)W).total;
    return total > 256 ? total : 256;           // > 0 also without polygons: 0 means refused
}

int mr_db_targets(const void *polygons, int dtype, const unsigned char *ignore_tags, const int *offsets, int N, int H, int W,
                  int capacity, double shrink_k, double min_text_size, float thresh_scale, float thresh_min, void *workspace,
                  int64_t workspace_bytes, float *gt, float *mask, float *thresh_map, float *thresh_mask, void *polygons_out,
                  unsigned char *ignore_out, int *status, void *stream) {
    if (bad_sizes(N, H, W, capacity) || (dtype != 0 && dtype != 1)) return MR_ERR_BAD_SHAPE;
    if (!offsets || !workspace || !gt || !mask || !thresh_map || !thresh_mask) return MR_ERR_NULL_POINTER;
    if (capacity > 0 && (!polygons || !ignore_tags || !polygons_out || !ignore_out || !status)) return MR_ERR_NULL_POINTER;
    const Layout l = layout(capacity, H, W);
    if (workspace_bytes < l.total) return MR_ERR_BAD_SHAPE;
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    SlotInfo *info = (SlotInfo *)(ws + l.o_info);
    int *slots = (int *)(ws + l.o_slots);
    int rc;
    const int64_t total = (int64_t)N * H * W;
    db_maps_init_kernel<<<(int)std::min<int64_t>(ceil_div(total, 256), 8192), 256, 0, st>>>(total, gt, mask, thresh_map, thresh_mask);
    if ((rc = check_launch("db_targets init"))) return rc;
    if (capacity > 0) {
        const int tb = (int)ceil_div(capacity, 64);
        if (dtype == 0)
            db_polygon_kernel<float><<<tb, 64, 0, st>>>((const float *)polygons, ignore_tags, offsets, N, H, W, capacity, shrink_k,
                                                        min_text_size, l.s, slots, info, (float *)polygons_out, ignore_out, status);
        else
            db_polygon_kernel<double><<<tb, 64, 0, st>>>((const double *)polygons, ignore_tags, offsets, N, H, W, capacity, shrink_k,
                                                         min_text_size, l.s, slots, info, (double *)polygons_out, ignore_out, status);
        if ((rc = check_launch("db_targets polygons"))) return rc;
        db_fill_kernel<<<dim3(capacity, 3), 256, 0, st>>>(info, slots, l.s, H, W, (mr_dbtgt::PolyEdge *)(ws + l.o_edges), gt, mask,
                                                          thresh_mask);
        if ((rc = check_launch("db_targets fill"))) return rc;
        if (dtype == 0)
            db_border_kernel<float><<<dim3(capacity, kBorderBands), 256, 0, st>>>(info, (const float *)polygons_out, H, W, thresh_map);
        else
            db_border_kernel<double><<<dim3(capacity, kBorderBands), 256, 0, st>>>(info, (const double *)polygons_out, H, W, thresh_map);
        if ((rc = check_launch("db_targets border"))) return rc;
    }
    db_thresh_scale_kernel<<<(int)std::min<int64_t>(ceil_div(total, 256), 8192), 256, 0, st>>>(total, thresh_scale, thresh_min,
                                                                                              thresh_map);
    return check_launch("db_targets scale");
}

}  // extern "C"
