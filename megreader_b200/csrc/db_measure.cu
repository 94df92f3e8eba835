// The DB detector's validation measure on the device: QuadMeasurer.measure (structure/measurers/quad_measurer.py), i.e.
// DetectionIoUEvaluator.evaluate_image (concern/icdar2015_eval/detection/iou.py:13-179) for every image of a batch.
//   1. db_measure_slot_kernel: one thread per gt slot and per det slot: the image of the slot, validity, GEOS area,
//      bounding box and convex pieces (db_measure_core.cuh); resets the per-slot outputs;
//   2. db_measure_pair_kernel: one thread per (gt slot, det) pair of the same image: the IoU in float64, and for a don't-care
//      gt the test intersection / area(det) > area_precision_constraint, which flags the det as don't-care (a boolean: the
//      reference's `break` at the first such gt changes nothing);
//   3. db_measure_image_kernel: one block per image: the indices among the image's valid polygons (block scans), the greedy
//      match in the reference's order (for each care gt in turn, the lowest-index unmatched care det with IoU above
//      iou_constraint, found with a block min-reduction over the det row), the counts, precision / recall / hmean, and the
//      optional int64 totals (care gt, care det, matched) that combine_results needs across batches.
// Inputs are packed with device offsets and counts, and no step reads anything back to the host, so a captured graph
// replays with new contents.  Bad offsets or counts are reported per image in `status` (such an image adds nothing to
// the totals), never by a fault.
#include "common.cuh"
#include "db_measure_core.cuh"

using namespace mr;
using mr_dbmeas::Ring;

namespace {

constexpr int kImageThreads = 256;

int64_t r256(int64_t b) { return round_up(b, 256); }

struct Layout {
    int64_t o_gt, o_det, o_gimg, o_iou, total;
};

Layout layout(int64_t N, int64_t cap, int64_t maxd) {
    Layout l;
    int64_t o = 0;
    l.o_gt = o;   o += r256(cap * (int64_t)sizeof(Ring));
    l.o_det = o;  o += r256(N * maxd * (int64_t)sizeof(Ring));
    l.o_gimg = o; o += r256(cap * 4);
    l.o_iou = o;  o += r256(cap * maxd * 8);
    l.total = o;
    return l;
}

__device__ __forceinline__ int clamp_off(int v, int cap) { return v < 0 ? 0 : v > cap ? cap : v; }

template <class TG, class TD>
__global__ void db_measure_slot_kernel(const TG *__restrict__ gt, const int *__restrict__ offsets, int N, int cap,
                                       const TD *__restrict__ det, const int *__restrict__ count, int maxd, Ring *gt_ring,
                                       Ring *det_ring, int *gt_image, int *gt_index, int *gt_match, int *det_index,
                                       unsigned char *det_dontcare, int *det_match) {
    const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t ndet = (int64_t)N * maxd;
    if (p >= cap + ndet) return;
    double q[8];
    Ring r;
    if (p < cap) {
        // image of the slot: the last n with offsets[n] <= p (offsets clamped to [0, cap]; empty images are skipped); slots
        // before offsets[0] or from offsets[N] on belong to no image
        int image = -1;
        if (p >= clamp_off(offsets[0], cap) && p < clamp_off(offsets[N], cap)) {
            int lo = 0, hi = N - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (clamp_off(offsets[mid], cap) <= p) lo = mid; else hi = mid - 1;
            }
            image = lo;
        }
        for (int k = 0; k < 8; ++k) q[k] = (double)gt[8 * p + k];
        r = mr_dbmeas::ring_prepare(q);
        if (image < 0) r.valid = 0;
        gt_ring[p] = r;
        gt_image[p] = image;
        gt_index[p] = -1;
        gt_match[p] = -1;
    } else {
        const int64_t d = p - cap;
        const int n = (int)(d / maxd), j = (int)(d % maxd);
        const int c = count[n];
        for (int k = 0; k < 8; ++k) q[k] = (double)det[8 * d + k];
        r = mr_dbmeas::ring_prepare(q);
        if (j >= c) r.valid = 0;
        det_ring[d] = r;
        det_index[d] = -1;
        det_dontcare[d] = 0;
        det_match[d] = -1;
    }
}

__global__ void db_measure_pair_kernel(const Ring *__restrict__ gt_ring, const Ring *__restrict__ det_ring,
                                       const int *__restrict__ gt_image, const unsigned char *__restrict__ tags, int cap, int maxd,
                                       double area_precision_constraint, double *iou, unsigned char *det_dontcare) {
    const int64_t total = (int64_t)cap * maxd;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t g = i / maxd;
        const int j = (int)(i % maxd);
        double v = 0.;
        const int n = gt_image[g];
        if (n >= 0 && gt_ring[g].valid) {
            const int64_t d = (int64_t)n * maxd + j;
            if (det_ring[d].valid) {
                double prec;
                mr_dbmeas::iou_precision(gt_ring[g], det_ring[d], &v, &prec);
                if (tags[g] && prec > area_precision_constraint) det_dontcare[d] = 1;
            }
        }
        iou[i] = v;
    }
}

// exclusive prefix count of flag over the block (blockDim.x == kImageThreads); *total the block's count
__device__ int block_scan(bool flag, int *warp_sums, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned ballot = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) warp_sums[warp] = __popc(ballot);
    __syncthreads();
    int before = 0, all = 0;
    for (int w = 0; w < kImageThreads / 32; ++w) {
        before += w < warp ? warp_sums[w] : 0;
        all += warp_sums[w];
    }
    __syncthreads();
    *total = all;
    return before + __popc(ballot & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(kImageThreads)
db_measure_image_kernel(const Ring *__restrict__ gt_ring, const Ring *__restrict__ det_ring, const int *__restrict__ gt_image,
                        const unsigned char *__restrict__ tags, const int *__restrict__ offsets, const int *__restrict__ count,
                        int cap, int maxd, double iou_constraint, const double *__restrict__ iou, int *gt_index, int *gt_match,
                        int *det_index, const unsigned char *__restrict__ det_dontcare, int *det_match, int *image_counts,
                        double *image_metrics, int *image_status, unsigned long long *totals) {
    __shared__ int warp_sums[kImageThreads / 32];
    __shared__ int best;
    const int n = blockIdx.x, tid = threadIdx.x;
    const int o0 = offsets[n], o1 = offsets[n + 1], c_in = count[n];
    const int status = (o0 < 0 || o1 < o0 || o1 > cap ? 1 : 0) | (c_in < 0 || c_in > maxd ? 2 : 0);
    const int lo = clamp_off(o0, cap), hi = max(lo, clamp_off(o1, cap));
    const int c = c_in < 0 ? 0 : c_in > maxd ? maxd : c_in;
    const int64_t dbase = (int64_t)n * maxd;

    // indices among the image's valid polygons, and the don't-care counts
    int gt_valid = 0, gt_dc = 0, det_valid = 0, det_dc = 0;
    for (int base = lo; base < hi; base += kImageThreads) {
        const int g = base + tid;
        const bool v = g < hi && gt_ring[g].valid && gt_image[g] == n;
        int chunk;
        const int idx = block_scan(v, warp_sums, &chunk);
        if (v) gt_index[g] = gt_valid + idx;
        gt_valid += chunk;
        gt_dc += __syncthreads_count(v && tags[g]);
    }
    for (int base = 0; base < c; base += kImageThreads) {
        const int j = base + tid;
        const bool v = j < c && det_ring[dbase + j].valid;
        int chunk;
        const int idx = block_scan(v, warp_sums, &chunk);
        if (v) det_index[dbase + j] = det_valid + idx;
        det_valid += chunk;
        det_dc += __syncthreads_count(v && det_dontcare[dbase + j]);
    }

    // greedy match, in the reference's order
    int matched = 0;
    for (int g = lo; g < hi; ++g) {
        // read-only inputs, so the branch is uniform over the block
        if (gt_image[g] != n || !gt_ring[g].valid || tags[g]) continue;
        if (tid == 0) best = 0x7fffffff;
        __syncthreads();
        const double *row = iou + (int64_t)g * maxd;
        int mine = 0x7fffffff;
        for (int j = tid; j < c; j += kImageThreads) {
            const int64_t d = dbase + j;
            if (row[j] > iou_constraint && det_index[d] >= 0 && !det_dontcare[d] && det_match[d] < 0) { mine = j; break; }
        }
        for (int s = 16; s > 0; s >>= 1) mine = min(mine, __shfl_xor_sync(0xffffffffu, mine, s));
        if ((tid & 31) == 0 && mine != 0x7fffffff) atomicMin(&best, mine);
        __syncthreads();
        const int b = best;
        if (b != 0x7fffffff) {
            if (tid == 0) {
                det_match[dbase + b] = gt_index[g];
                gt_match[g] = det_index[dbase + b];
            }
            ++matched;
        }
        __syncthreads();
    }

    if (tid == 0) {
        const int gt_care = gt_valid - gt_dc, det_care = det_valid - det_dc;
        int *cnt = image_counts + 5 * (int64_t)n;
        cnt[0] = gt_care; cnt[1] = det_care; cnt[2] = matched; cnt[3] = gt_valid; cnt[4] = det_valid;
        double *m = image_metrics + 3 * (int64_t)n;
        mr_dbmeas::image_metrics(gt_care, det_care, matched, m, m + 1, m + 2);
        image_status[n] = status;
        if (totals && status == 0) {
            atomicAdd(totals, (unsigned long long)gt_care);
            atomicAdd(totals + 1, (unsigned long long)det_care);
            atomicAdd(totals + 2, (unsigned long long)matched);
        }
    }
}

bool bad_sizes(int64_t N, int64_t cap, int64_t maxd) {
    return N <= 0 || N > ((int64_t)1 << 24) || cap < 0 || cap > ((int64_t)1 << 24) || maxd < 0 || maxd > ((int64_t)1 << 20) ||
           N * maxd > ((int64_t)1 << 28) || cap * maxd > ((int64_t)1 << 32);
}

template <class TG, class TD>
void launch_slots(const void *gt, const int *offsets, int N, int cap, const void *det, const int *count, int maxd, Ring *gr, Ring *dr,
                  int *gimg, int *gt_index, int *gt_match, int *det_index, unsigned char *det_dc, int *det_match, cudaStream_t st) {
    const int64_t slots = cap + (int64_t)N * maxd;
    db_measure_slot_kernel<TG, TD><<<(unsigned)ceil_div(slots, 128), 128, 0, st>>>((const TG *)gt, offsets, N, cap, (const TD *)det,
                                                                                 count, maxd, gr, dr, gimg, gt_index, gt_match,
                                                                                 det_index, det_dc, det_match);
}

}  // namespace

extern "C" {

int64_t mr_db_measure_workspace_bytes(int64_t N, int64_t capacity, int64_t max_dets) {
    if (bad_sizes(N, capacity, max_dets)) return 0;
    const int64_t total = layout(N, capacity, max_dets).total;
    return total > 256 ? total : 256;           // > 0 also without polygons: 0 means refused
}

int mr_db_measure(const void *gt_polygons, int gt_dtype, const unsigned char *ignore_tags, const int *offsets, int N, int capacity,
                  const void *boxes, int det_dtype, const int *count, int max_dets, double iou_constraint,
                  double area_precision_constraint, void *workspace, int64_t workspace_bytes, int *gt_index, int *gt_match,
                  int *det_index, unsigned char *det_dontcare, int *det_match, int *image_counts, double *image_metrics,
                  int *image_status, double *iou, long long *totals, void *stream) {
    if (bad_sizes(N, capacity, max_dets) || (gt_dtype != 0 && gt_dtype != 1) || (det_dtype != 0 && det_dtype != 1))
        return MR_ERR_BAD_SHAPE;
    if (!offsets || !count || !workspace || !image_counts || !image_metrics || !image_status) return MR_ERR_NULL_POINTER;
    if (capacity > 0 && (!gt_polygons || !ignore_tags || !gt_index || !gt_match)) return MR_ERR_NULL_POINTER;
    if (max_dets > 0 && (!boxes || !det_index || !det_dontcare || !det_match)) return MR_ERR_NULL_POINTER;
    const Layout l = layout(N, capacity, max_dets);
    if (workspace_bytes < l.total) return MR_ERR_BAD_SHAPE;
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    Ring *gr = (Ring *)(ws + l.o_gt), *dr = (Ring *)(ws + l.o_det);
    int *gimg = (int *)(ws + l.o_gimg);
    double *iou_buf = iou ? iou : (double *)(ws + l.o_iou);
    int rc;
    if (capacity + (int64_t)N * max_dets > 0) {
        if (gt_dtype == 0 && det_dtype == 0)
            launch_slots<float, int>(gt_polygons, offsets, N, capacity, boxes, count, max_dets, gr, dr, gimg, gt_index, gt_match,
                                     det_index, det_dontcare, det_match, st);
        else if (gt_dtype == 0)
            launch_slots<float, double>(gt_polygons, offsets, N, capacity, boxes, count, max_dets, gr, dr, gimg, gt_index, gt_match,
                                        det_index, det_dontcare, det_match, st);
        else if (det_dtype == 0)
            launch_slots<double, int>(gt_polygons, offsets, N, capacity, boxes, count, max_dets, gr, dr, gimg, gt_index, gt_match,
                                      det_index, det_dontcare, det_match, st);
        else
            launch_slots<double, double>(gt_polygons, offsets, N, capacity, boxes, count, max_dets, gr, dr, gimg, gt_index,
                                         gt_match, det_index, det_dontcare, det_match, st);
        if ((rc = check_launch("db_measure slots"))) return rc;
    }
    const int64_t pairs = (int64_t)capacity * max_dets;
    if (pairs > 0) {
        db_measure_pair_kernel<<<(unsigned)std::min<int64_t>(ceil_div(pairs, 256), 65536), 256, 0, st>>>(
            gr, dr, gimg, ignore_tags, capacity, max_dets, area_precision_constraint, iou_buf, det_dontcare);
        if ((rc = check_launch("db_measure pairs"))) return rc;
    }
    db_measure_image_kernel<<<N, kImageThreads, 0, st>>>(gr, dr, gimg, ignore_tags, offsets, count, capacity, max_dets,
                                                         iou_constraint, iou_buf, gt_index, gt_match, det_index, det_dontcare,
                                                         det_match, image_counts, image_metrics, image_status,
                                                         (unsigned long long *)totals);
    return check_launch("db_measure image");
}

}  // extern "C"
