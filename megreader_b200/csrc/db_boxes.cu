// SegDetectorRepresenter on the device (structure/representers/seg_detector_representer.py:60-123):
//   bitmap = dest > thresh;  contours = cv2.findContours(bitmap, RETR_LIST, CHAIN_APPROX_NONE);  contours[:max_candidates]
// with the contours' points in cv2's order (the per-candidate geometry depends on it), then per kept contour get_mini_boxes,
// box_score_fast, the unclip, the second get_mini_boxes and the rescale.
//
// cv2's list is one contour per 8-connected foreground component (outer border, starting at the component's first raster
// pixel) and one per 4-connected background component that does not touch the frame (hole border, starting at the foreground
// pixel left of the hole's first raster pixel), in DESCENDING raster order of the start pixels.  So:
//   1. binarize, and label both classes by union-find in which a root always links to the smaller linear index: each root is
//      its component's first raster pixel, whatever the scheduling;
//   2. flag the background components that touch the frame;
//   3. mark the start pixels and give each its cv2 index by an exclusive count in reverse raster order; the first
//      max_candidates are kept (the reference truncates before any filtering);
//   4. trace every kept border (db_boxes_core.cuh), once to count its points and once to write them at scanned offsets;
//   5. (mr_db_box_candidates_f32) one thread per kept contour: convex hull, rotating calipers, box corners, masked mean;
//   6. (mr_db_boxes_f32, all of the above plus) one thread per candidate: box_thresh, unclip, second box, rescale; then the
//      survivors compacted per image in candidate order.
// No host synchronisation: every entry can be captured in a CUDA graph.
#include <cub/cub.cuh>

#include "common.cuh"
#include "db_boxes_core.cuh"

using namespace mr;

namespace {

constexpr int kChunk = 1024;            // pixels per block of the start-count / rank passes (= threads per block)
constexpr int kMinSize = 3;             // SegDetectorRepresenter.min_size (seg_detector_representer.py:21)
// pixels per image: the int32 point offsets must hold the points of an image (a pixel is passed at most 8 times)
constexpr int64_t kMaxPixels = ((int64_t)1 << 28) - 1;

int64_t r256(int64_t b) { return round_up(b, 256); }

struct Workspace {
    unsigned char *bm, *frame;
    int *lab, *chunk, *cand, *len;
};

int64_t chunks_of(int64_t HW) { return ceil_div(HW, kChunk); }

int64_t workspace_bytes(int64_t N, int64_t HW, int64_t maxc) {
    return 2 * r256(N * HW) + r256(4 * N * HW) + r256(4 * N * chunks_of(HW)) + 2 * r256(4 * N * maxc);
}

Workspace carve(void *ws, int64_t N, int64_t HW, int64_t maxc) {
    char *p = (char *)ws;
    Workspace w;
    w.bm = (unsigned char *)p;                        p += r256(N * HW);
    w.frame = (unsigned char *)p;                     p += r256(N * HW);
    w.lab = (int *)p;                                 p += r256(4 * N * HW);
    w.chunk = (int *)p;                               p += r256(4 * N * chunks_of(HW));
    w.cand = (int *)p;                                p += r256(4 * N * maxc);
    w.len = (int *)p;
    return w;
}

__global__ void db_binarize_kernel(const float *__restrict__ dest, int64_t total, int HW, float thresh, unsigned char *bm,
                                   unsigned char *frame, int *lab) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        bm[i] = dest[i] > thresh;
        frame[i] = 0;
        lab[i] = (int)(i % HW);
    }
}

__device__ __forceinline__ int uf_find(const volatile int *L, int x) {
    int p = L[x];
    while (p != x) {
        x = p;
        p = L[x];
    }
    return x;
}

// links the trees of a and b; the larger root is pointed at the smaller one, retried until the link holds
__device__ void uf_unite(volatile int *L, int a, int b) {
    for (;;) {
        a = uf_find(L, a);
        b = uf_find(L, b);
        if (a == b) return;
        if (a > b) { const int t = a; a = b; b = t; }
        const int old = atomicMin((int *)&L[b], a);
        if (old == b) return;
        b = old;
    }
}

// foreground: 8-connectivity, background: 4-connectivity (the backward half of each neighbourhood)
__global__ void db_label_union_kernel(const unsigned char *__restrict__ bm, int *lab, int64_t total, int H, int W) {
    const int HW = H * W;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t base = i - i % HW;
        const unsigned char *b = bm + base;
        volatile int *L = lab + base;
        const int p = (int)(i - base), x = p % W, y = p / W;
        const unsigned char v = b[p];
        if (x > 0 && b[p - 1] == v) uf_unite(L, p, p - 1);
        if (y > 0) {
            if (b[p - W] == v) uf_unite(L, p, p - W);
            if (v) {
                if (x > 0 && b[p - W - 1]) uf_unite(L, p, p - W - 1);
                if (x < W - 1 && b[p - W + 1]) uf_unite(L, p, p - W + 1);
            }
        }
    }
}

__global__ void db_label_flatten_kernel(const unsigned char *__restrict__ bm, int *lab, unsigned char *frame, int64_t total, int H,
                                        int W) {
    const int HW = H * W;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t base = i - i % HW;
        const int p = (int)(i - base), x = p % W, y = p / W;
        const int r = uf_find(lab + base, p);
        lab[i] = r;
        if (!bm[i] && (x == 0 || y == 0 || x == W - 1 || y == H - 1)) frame[base + r] = 1;
    }
}

// 0: no contour starts at q; 1: an outer border does (q is a foreground root); 2: a hole border does (q + 1 is the root of a
// background component off the frame -- a root in column 0 is on the frame, so q + 1 never wraps to the next row).  The two
// never coincide: the pixel above a hole's first pixel is foreground and 8-adjacent to q, and comes first in raster order.
__device__ __forceinline__ int start_kind(const unsigned char *b, const int *L, const unsigned char *F, int q, int HW) {
    if (q >= HW || !b[q]) return 0;
    if (L[q] == q) return 1;
    return (q + 1 < HW && !b[q + 1] && L[q + 1] == q + 1 && !F[q + 1]) ? 2 : 0;
}

using BlockScan = cub::BlockScan<int, kChunk>;

__global__ void __launch_bounds__(kChunk) db_start_count_kernel(Workspace w, int HW, int nchunks) {
    using Reduce = cub::BlockReduce<int, kChunk>;
    __shared__ typename Reduce::TempStorage tmp;
    const int64_t base = (int64_t)blockIdx.y * HW;
    const int q = blockIdx.x * kChunk + threadIdx.x;
    const int f = start_kind(w.bm + base, w.lab + base, w.frame + base, q, HW) != 0;
    const int s = Reduce(tmp).Sum(f);
    if (threadIdx.x == 0) w.chunk[(int64_t)blockIdx.y * nchunks + blockIdx.x] = s;
}

// per image: chunk counts -> number of starts in later chunks (in place); total[n] and count[n] = min(total, maxc)
__global__ void __launch_bounds__(kChunk) db_start_scan_kernel(Workspace w, int nchunks, int maxc, int *count, int *total) {
    __shared__ typename BlockScan::TempStorage tmp;
    int *c = w.chunk + (int64_t)blockIdx.x * nchunks;
    int carry = 0;
    for (int hi = nchunks; hi > 0; hi -= kChunk) {
        const int j = hi - 1 - (int)threadIdx.x;
        const int v = j >= 0 ? c[j] : 0;
        int ex, agg;
        BlockScan(tmp).ExclusiveSum(v, ex, agg);
        if (j >= 0) c[j] = carry + ex;
        carry += agg;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        total[blockIdx.x] = carry;
        count[blockIdx.x] = carry < maxc ? carry : maxc;
    }
}

// cv2 index of every start = starts after it in raster order; the first maxc are kept as 2 * q + (hole border)
__global__ void __launch_bounds__(kChunk) db_start_rank_kernel(Workspace w, int HW, int nchunks, int maxc) {
    __shared__ typename BlockScan::TempStorage tmp;
    const int64_t base = (int64_t)blockIdx.y * HW;
    const int q = blockIdx.x * kChunk + (kChunk - 1 - (int)threadIdx.x);
    const int k = start_kind(w.bm + base, w.lab + base, w.frame + base, q, HW);
    int ex;
    BlockScan(tmp).ExclusiveSum(k != 0, ex);
    const int rank = w.chunk[(int64_t)blockIdx.y * nchunks + blockIdx.x] + ex;
    if (k && rank < maxc) w.cand[(int64_t)blockIdx.y * maxc + rank] = 2 * q + (k == 2);
}

__global__ void db_trace_count_kernel(Workspace w, int N, int H, int W, int maxc, const int *count) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * maxc) return;
    const int n = (int)(i / maxc), c = (int)(i % maxc);
    if (c >= count[n]) return;
    const int code = w.cand[i], q = code >> 1;
    w.len[i] = mr_dbbox::trace_border(w.bm + (int64_t)n * H * W, H, W, q % W, q / W, code & 1, [](int, int) {});
}

// per image: offsets[n][c] = first point of contour c; entries past count[n] hold the image's number of points
__global__ void __launch_bounds__(kChunk) db_trace_offsets_kernel(Workspace w, int maxc, const int *count, int *offsets) {
    __shared__ typename BlockScan::TempStorage tmp;
    const int n = blockIdx.x, cnt = count[n];
    const int *len = w.len + (int64_t)n * maxc;
    int *off = offsets + (int64_t)n * (maxc + 1);
    if (threadIdx.x == 0) off[0] = 0;
    int carry = 0;
    for (int lo = 0; lo < maxc; lo += kChunk) {
        const int c = lo + threadIdx.x;
        const int v = c < cnt ? len[c] : 0;
        int in, agg;
        BlockScan(tmp).InclusiveSum(v, in, agg);
        if (c < maxc) off[c + 1] = carry + in;
        carry += agg;
        __syncthreads();
    }
}

__global__ void db_trace_write_kernel(Workspace w, int N, int H, int W, int maxc, const int *count, const int *offsets,
                                      int *points, int64_t capacity) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * maxc) return;
    const int n = (int)(i / maxc), c = (int)(i % maxc);
    if (c >= count[n]) return;
    const int code = w.cand[i], q = code >> 1;
    int64_t k = offsets[(int64_t)n * (maxc + 1) + c];
    int *pts = points + (int64_t)n * capacity * 2;
    mr_dbbox::trace_border(w.bm + (int64_t)n * H * W, H, W, q % W, q / W, code & 1, [&](int x, int y) {
        if (k < capacity) {
            pts[2 * k] = x;
            pts[2 * k + 1] = y;
        }
        ++k;
    });
}

// The per-candidate steps before the unclip (seg_detector_representer.py:81-96) for every kept contour: get_mini_boxes
// (:125-145: cv::convexHull -> cv::minAreaRect -> cv::boxPoints -> the reference's corner order), and where sside >= min_size
// box_score_fast (:156-168) on the score map.  Scratch of contour c with n points: 6 n + 2 words at 6 offsets[c] + 2 c.
__global__ void db_box_candidate_kernel(const int *points, int64_t capacity, const int *offsets, const int *count,
                                        const float *binary, int N, int H, int W, int maxc, int *scratch, float *boxes,
                                        float *ssides, double *scores) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * maxc) return;
    const int n = (int)(i / maxc), c = (int)(i % maxc);
    float *box = boxes + i * 8;
    const int *off = offsets + (int64_t)n * (maxc + 1);
    const int64_t end = off[c + 1];
    scores[i] = 0.;
    if (c >= count[n] || end > capacity) {            // no contour, or one whose points did not fit
        for (int k = 0; k < 8; ++k) box[k] = 0.f;
        ssides[i] = c >= count[n] ? 0.f : -1.f;
        return;
    }
    const int len = (int)(end - off[c]);
    const mr_dbbox::Pt *p = (const mr_dbbox::Pt *)(points + ((int64_t)n * capacity + off[c]) * 2);
    int *s = scratch + (int64_t)n * (6 * capacity + 2 * maxc) + 6 * (int64_t)off[c] + 2 * c;
    int *o = s, *stack = s + len, *hull = s + 2 * len + 2;
    const int k = mr_dbbox::convex_hull(p, len, o, stack, hull);
    float *qx = (float *)s, *qy = qx + k, *vx = (float *)(s + 3 * len + 2), *vy = vx + k, *inv = vy + k;
    for (int j = 0; j < k; ++j) {                    // o and stack are free now; hull lies past 2 k floats
        const mr_dbbox::Pt q = p[hull[j]];
        qx[j] = (float)q.x;
        qy[j] = (float)q.y;
    }
    const mr_dbbox::Rect r = mr_dbbox::min_area_rect_hull(qx, qy, k, vx, vy, inv);
    const float sside = mr_dbbox::mini_box(r, box);
    ssides[i] = sside;
    if (sside >= (float)kMinSize) scores[i] = mr_dbbox::box_score(binary + (int64_t)n * H * W, H, W, box);
}

// The candidate loop after the score (seg_detector_representer.py:95-111) for every candidate: box_thresh, unclip, the second
// get_mini_boxes, sside >= min_size + 2 and the rescale to the destination size.  One thread per candidate; scratch of
// 8 K + 2 words per candidate for the offset path (K points at most) and the second hull.
__global__ void db_unclip_box_kernel(const float *boxes, const float *ssides, const double *scores, int N, int H, int W, int maxc,
                                     double box_thresh, const int *dest_sizes, int K, int *scratch, int *ibox, int *keep) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * maxc) return;
    keep[i] = 0;
    if (!(ssides[i] >= (float)kMinSize) || box_thresh > scores[i]) return;
    const float *box = boxes + i * 8;
    const double delta = mr_dbbox::unclip_distance(box);
    if (mr_dbbox::unclip_max_points(delta) > K) { keep[i] = -1; return; }    // larger than any box of this map size
    int *s = scratch + i * (8 * (int64_t)K + 2);
    int *px = s, *py = s + K;
    const int n = mr_dbbox::unclip_offset(box, delta, px, py, K);
    if (n <= 0) { keep[i] = n < 0 ? -1 : 0; return; }
    mr_dbbox::Pt *pt = (mr_dbbox::Pt *)(s + 6 * K + 2);             // interleave after the hull scratch
    for (int j = 0; j < n; ++j) pt[j] = mr_dbbox::Pt{px[j], py[j]};
    int *o = s, *stack = s + K, *hull = s + 2 * K + 2;               // the offset path now lives in pt
    const int k = mr_dbbox::convex_hull(pt, n, o, stack, hull);
    float *qx = (float *)(s + 3 * K + 2), *qy = qx + k, *vx = (float *)s, *vy = vx + k, *inv = vy + k;
    for (int j = 0; j < k; ++j) {
        qx[j] = (float)pt[hull[j]].x;
        qy[j] = (float)pt[hull[j]].y;
    }
    const mr_dbbox::Rect r = mr_dbbox::min_area_rect_hull(qx, qy, k, vx, vy, inv);
    float b2[8];
    if (mr_dbbox::mini_box(r, b2) < (float)(kMinSize + 2)) return;
    const int n_img = (int)(i / maxc);
    const int dh = dest_sizes ? dest_sizes[2 * n_img] : H, dw = dest_sizes ? dest_sizes[2 * n_img + 1] : W;
    for (int j = 0; j < 4; ++j) {
        ibox[i * 8 + 2 * j] = mr_dbbox::rescale(b2[2 * j], W, dw);
        ibox[i * 8 + 2 * j + 1] = mr_dbbox::rescale(b2[2 * j + 1], H, dh);
    }
    keep[i] = 1;
}

// per image: the kept boxes in candidate order -> out_boxes [N, maxc, 4, 2], out_scores [N, maxc] (zero past count[n])
__global__ void __launch_bounds__(kChunk) db_compact_kernel(const int *ibox, const int *keep, const double *scores, int maxc,
                                                            int *out_boxes, float *out_scores, int *count) {
    __shared__ typename BlockScan::TempStorage tmp;
    const int n = blockIdx.x;
    int carry = 0;
    for (int lo = 0; lo < maxc; lo += kChunk) {
        const int c = lo + threadIdx.x;
        const int64_t i = (int64_t)n * maxc + c;
        const int k = c < maxc && keep[i] == 1;
        int ex, agg;
        BlockScan(tmp).ExclusiveSum(k, ex, agg);
        if (k) {
            const int64_t o = (int64_t)n * maxc + carry + ex;
            for (int j = 0; j < 8; ++j) out_boxes[o * 8 + j] = ibox[i * 8 + j];
            out_scores[o] = (float)scores[i];
        }
        carry += agg;
        __syncthreads();
    }
    for (int c = carry + (int)threadIdx.x; c < maxc; c += kChunk) {
        const int64_t o = (int64_t)n * maxc + c;
        for (int j = 0; j < 8; ++j) out_boxes[o * 8 + j] = 0;
        out_scores[o] = 0.f;
    }
    if (threadIdx.x == 0) count[n] = carry;
}

int elem_blocks(int64_t n) { return (int)std::min<int64_t>(ceil_div(n, 256), 8 * (int64_t)sm_count()); }

}  // namespace

extern "C" {

int64_t mr_db_contours_workspace_bytes(int64_t N, int64_t H, int64_t W, int64_t max_candidates) {
    if (N <= 0 || N > 65535 || H <= 0 || W <= 0 || max_candidates < 0 || H * W > kMaxPixels) return 0;
    return workspace_bytes(N, H * W, max_candidates);
}

int mr_db_contours_f32(const float *dest, int N, int H, int W, float thresh, int max_candidates, void *workspace,
                       int64_t workspace_bytes_given, int *points, int64_t point_capacity, int *offsets, int *count, int *total,
                       void *stream) {
    if (N < 0 || N > 65535 || max_candidates < 0 || point_capacity < 0) return MR_ERR_BAD_SHAPE;   // N is a grid y dimension
    if (N == 0) return MR_OK;
    if (H <= 0 || W <= 0 || (int64_t)H * W > kMaxPixels) return MR_ERR_BAD_SHAPE;
    if (!dest || !workspace || !offsets || !count || !total || (point_capacity > 0 && !points)) return MR_ERR_NULL_POINTER;
    const int HW = H * W;
    if (workspace_bytes_given < workspace_bytes(N, HW, max_candidates)) return MR_ERR_BAD_SHAPE;
    cudaStream_t st = (cudaStream_t)stream;
    const Workspace w = carve(workspace, N, HW, max_candidates);
    const int64_t px = (int64_t)N * HW;
    const int nchunks = (int)chunks_of(HW);
    int rc;
    db_binarize_kernel<<<elem_blocks(px), 256, 0, st>>>(dest, px, HW, thresh, w.bm, w.frame, w.lab);
    if ((rc = check_launch("db_contours binarize"))) return rc;
    db_label_union_kernel<<<elem_blocks(px), 256, 0, st>>>(w.bm, w.lab, px, H, W);
    if ((rc = check_launch("db_contours union"))) return rc;
    db_label_flatten_kernel<<<elem_blocks(px), 256, 0, st>>>(w.bm, w.lab, w.frame, px, H, W);
    if ((rc = check_launch("db_contours flatten"))) return rc;
    db_start_count_kernel<<<dim3(nchunks, N), kChunk, 0, st>>>(w, HW, nchunks);
    if ((rc = check_launch("db_contours start count"))) return rc;
    db_start_scan_kernel<<<N, kChunk, 0, st>>>(w, nchunks, max_candidates, count, total);
    if ((rc = check_launch("db_contours start scan"))) return rc;
    const int tb = (int)ceil_div((int64_t)N * max_candidates, 128);
    if (max_candidates > 0) {
        db_start_rank_kernel<<<dim3(nchunks, N), kChunk, 0, st>>>(w, HW, nchunks, max_candidates);
        if ((rc = check_launch("db_contours start rank"))) return rc;
        db_trace_count_kernel<<<tb, 128, 0, st>>>(w, N, H, W, max_candidates, count);
        if ((rc = check_launch("db_contours trace count"))) return rc;
    }
    db_trace_offsets_kernel<<<N, kChunk, 0, st>>>(w, max_candidates, count, offsets);
    if ((rc = check_launch("db_contours offsets"))) return rc;
    if (max_candidates == 0) return MR_OK;
    db_trace_write_kernel<<<tb, 128, 0, st>>>(w, N, H, W, max_candidates, count, offsets, points, point_capacity);
    return check_launch("db_contours trace write");
}

int64_t mr_db_box_candidates_workspace_bytes(int64_t N, int64_t max_candidates, int64_t point_capacity) {
    if (N <= 0 || max_candidates < 0 || point_capacity < 0) return 0;
    return r256(4 * N * (6 * point_capacity + 2 * max_candidates));
}

int mr_db_box_candidates_f32(const int *points, int64_t point_capacity, const int *offsets, const int *count, const float *binary,
                             int N, int H, int W, int max_candidates, void *workspace, int64_t workspace_bytes_given, float *boxes,
                             float *ssides, double *scores, void *stream) {
    if (N < 0 || N > 65535 || max_candidates < 0 || point_capacity < 0 || point_capacity > INT32_MAX) return MR_ERR_BAD_SHAPE;
    if (N == 0 || max_candidates == 0) return MR_OK;
    if (H <= 0 || W <= 0 || (int64_t)H * W > kMaxPixels) return MR_ERR_BAD_SHAPE;
    if ((point_capacity > 0 && !points) || !offsets || !count || !binary || !workspace || !boxes || !ssides || !scores)
        return MR_ERR_NULL_POINTER;
    if (workspace_bytes_given < mr_db_box_candidates_workspace_bytes(N, max_candidates, point_capacity)) return MR_ERR_BAD_SHAPE;
    const int tb = (int)ceil_div((int64_t)N * max_candidates, 128);
    db_box_candidate_kernel<<<tb, 128, 0, (cudaStream_t)stream>>>(points, point_capacity, offsets, count, binary, N, H, W,
                                                                   max_candidates, (int *)workspace, boxes, ssides, scores);
    return check_launch("db_box_candidates");
}

}  // extern "C"

namespace {

// the point capacity mr_db_boxes_f32 gives find_contours, and the offset-path bound of its unclip scratch
int64_t boxes_capacity(int64_t H, int64_t W) { return 4 * H * W; }
int unclip_points(int64_t H, int64_t W) { return mr_dbbox::unclip_max_points(0.75 * (double)(H > W ? H : W) + 2.); }

struct BoxesLayout {
    int64_t contours_ws, cand_ws, total;
    int64_t o_points, o_offsets, o_count, o_total, o_cand, o_cboxes, o_ssides, o_scores, o_unclip, o_ibox, o_keep;
};

BoxesLayout boxes_layout(int64_t N, int64_t H, int64_t W, int64_t maxc) {
    BoxesLayout l;
    const int64_t cap = boxes_capacity(H, W), K = unclip_points(H, W), NC = N * maxc;
    l.contours_ws = workspace_bytes(N, H * W, maxc);
    l.cand_ws = r256(4 * N * (6 * cap + 2 * maxc));
    int64_t o = l.contours_ws;
    l.o_points = o;  o += r256(8 * N * cap);
    l.o_offsets = o; o += r256(4 * N * (maxc + 1));
    l.o_count = o;   o += r256(4 * N);
    l.o_total = o;   o += r256(4 * N);
    l.o_cand = o;    o += l.cand_ws;
    l.o_cboxes = o;  o += r256(32 * NC);
    l.o_ssides = o;  o += r256(4 * NC);
    l.o_scores = o;  o += r256(8 * NC);
    l.o_unclip = o;  o += r256(4 * NC * (8 * K + 2));
    l.o_ibox = o;    o += r256(32 * NC);
    l.o_keep = o;    o += r256(4 * NC);
    l.total = o;
    return l;
}

}  // namespace

extern "C" {

int64_t mr_db_boxes_workspace_bytes(int64_t N, int64_t H, int64_t W, int64_t max_candidates) {
    if (N <= 0 || N > 65535 || H <= 0 || W <= 0 || max_candidates < 0 || H * W > kMaxPixels) return 0;
    return boxes_layout(N, H, W, max_candidates).total;
}

int mr_db_boxes_f32(const float *binary, const float *dest, int N, int H, int W, float thresh, double box_thresh, int max_candidates,
                    const int *dest_sizes, void *workspace, int64_t workspace_bytes_given, int *boxes, float *scores, int *count,
                    void *stream) {
    if (N < 0 || N > 65535 || max_candidates < 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (H <= 0 || W <= 0 || (int64_t)H * W > kMaxPixels) return MR_ERR_BAD_SHAPE;
    if (!binary || !dest || !workspace || !boxes || !scores || !count) return MR_ERR_NULL_POINTER;
    const BoxesLayout l = boxes_layout(N, H, W, max_candidates);
    if (workspace_bytes_given < l.total) return MR_ERR_BAD_SHAPE;
    char *ws = (char *)workspace;
    const int64_t cap = boxes_capacity(H, W);
    int *points = (int *)(ws + l.o_points), *offsets = (int *)(ws + l.o_offsets), *cnt = (int *)(ws + l.o_count);
    int rc = mr_db_contours_f32(dest, N, H, W, thresh, max_candidates, ws, l.contours_ws, points, cap, offsets, cnt,
                                (int *)(ws + l.o_total), stream);
    if (rc) return rc;
    if (max_candidates == 0) {
        MR_CUDA_TRY(cudaMemsetAsync(count, 0, 4 * (size_t)N, (cudaStream_t)stream), "db_boxes count");
        return MR_OK;
    }
    float *cboxes = (float *)(ws + l.o_cboxes), *ssides = (float *)(ws + l.o_ssides);
    double *cscores = (double *)(ws + l.o_scores);
    rc = mr_db_box_candidates_f32(points, cap, offsets, cnt, binary, N, H, W, max_candidates, ws + l.o_cand, l.cand_ws, cboxes,
                                  ssides, cscores, stream);
    if (rc) return rc;
    const int K = unclip_points(H, W);
    const int tb = (int)ceil_div((int64_t)N * max_candidates, 128);
    int *ibox = (int *)(ws + l.o_ibox), *keep = (int *)(ws + l.o_keep);
    db_unclip_box_kernel<<<tb, 128, 0, (cudaStream_t)stream>>>(cboxes, ssides, cscores, N, H, W, max_candidates, box_thresh,
                                                                dest_sizes, K, (int *)(ws + l.o_unclip), ibox, keep);
    if ((rc = check_launch("db_boxes unclip"))) return rc;
    db_compact_kernel<<<N, kChunk, 0, (cudaStream_t)stream>>>(ibox, keep, cscores, max_candidates, boxes, scores, count);
    return check_launch("db_boxes compact");
}

}  // extern "C"
