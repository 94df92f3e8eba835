// Per-contour routines of SegDetectorRepresenter (structure/representers/seg_detector_representer.py:73-96, 125-168), shared by
// the CUDA kernels (db_boxes.cu) and by a host-side harness (tests/host_harness/db_boxes_core_host.cpp) that runs the SAME
// routines on the CPU against cv2: border following (cv2.findContours(RETR_LIST, CHAIN_APPROX_NONE)), convex hull and rotating
// calipers (cv2.minAreaRect), box corners (cv2.boxPoints + get_mini_boxes' order), quad fill (cv2.fillPoly) and the masked mean
// (cv2.mean).  Products and sums that must round as cv2's x86 build does (no fused multiply-add) go through fmul / fadd / dmul /
// dadd, which are __fmul_rn-style intrinsics on the device and plain operators on the host (built with -ffp-contract=off).
//
// The tracer is Suzuki-Abe border following as cv2 applies it: from the start pixel it looks for the first non-zero
// 8-neighbour turning from "left" (outer border) or "right" (hole border) in decreasing direction codes, then repeatedly
// scans the neighbours of the current pixel in increasing direction codes from the one after the pixel it came from,
// emitting the current pixel at every step, until it leaves the start pixel towards the first neighbour again.  Pixels on
// one-pixel-wide parts are therefore emitted once per pass.  Only "zero / non-zero" of the bitmap is read; outside the map
// counts as zero (cv2 pads the image with a zero frame).
//
// Direction codes (x right, y down): 0 = (+1, 0), 1 = (+1, -1), 2 = (0, -1), 3 = (-1, -1), 4 = (-1, 0), 5 = (-1, +1),
// 6 = (0, +1), 7 = (+1, +1).
#pragma once
#include <math.h>
#include <stdint.h>

#if !defined(__CUDACC__) && !defined(__host__)
#define __host__
#define __device__
#endif

namespace mr_dbbox {

__host__ __device__ inline int dir_dx(int s) { return (s == 0 || s == 1 || s == 7) ? 1 : (s >= 3 && s <= 5) ? -1 : 0; }
__host__ __device__ inline int dir_dy(int s) { return (s >= 1 && s <= 3) ? -1 : (s >= 5 && s <= 7) ? 1 : 0; }

__host__ __device__ inline bool on(const unsigned char *bm, int H, int W, int x, int y) {
    return x >= 0 && y >= 0 && x < W && y < H && bm[(int64_t)y * W + x] != 0;
}

// Traces the border that starts at (x0, y0): an outer border when `hole` is false (the start is the first raster pixel of an
// 8-connected foreground component), a hole border otherwise (the start is the foreground pixel left of the first raster
// pixel of an enclosed 4-connected background component).  Calls emit(x, y) for every contour point in cv2's order and
// returns their number.
template <class Emit>
__host__ __device__ inline int trace_border(const unsigned char *bm, int H, int W, int x0, int y0, bool hole, Emit emit) {
    int s = hole ? 0 : 4;
    const int s_first = s;
    int x1, y1;
    do {
        s = (s - 1) & 7;
        x1 = x0 + dir_dx(s);
        y1 = y0 + dir_dy(s);
    } while (!on(bm, H, W, x1, y1) && s != s_first);
    if (s == s_first) {                     // isolated pixel
        emit(x0, y0);
        return 1;
    }
    int n = 0, x3 = x0, y3 = y0;
    for (;;) {
        int x4, y4;
        do {                                // the pixel we came from is non-zero, so this stops within 8 steps
            ++s;
            x4 = x3 + dir_dx(s & 7);
            y4 = y3 + dir_dy(s & 7);
        } while (!on(bm, H, W, x4, y4));
        s &= 7;
        emit(x3, y3);
        ++n;
        if (x4 == x0 && y4 == y0 && x3 == x1 && y3 == y1) break;
        x3 = x4;
        y3 = y4;
        s = (s + 4) & 7;
    }
    return n;
}

}  // namespace mr_dbbox

namespace mr_dbbox {

// float products and sums that must round exactly as cv2's x86 build (no fused multiply-add) does
#ifdef __CUDA_ARCH__
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
#else
inline float fmul(float a, float b) { return a * b; }
inline float fadd(float a, float b) { return a + b; }
inline float fsub(float a, float b) { return a - b; }
inline double dmul(double a, double b) { return a * b; }
inline double dadd(double a, double b) { return a + b; }
inline double dsub(double a, double b) { return a - b; }
#endif

}  // namespace mr_dbbox

// ---- per-candidate geometry (seg_detector_representer.py:81-85, 125-145: get_mini_boxes = cv2.minAreaRect + cv2.boxPoints) ----
namespace mr_dbbox {

// A point of cv::convexHull's input: int (contours) or float (cv2.minAreaRect of float32 polygons)
template <class T> struct PtT { T x, y; };
using Pt = PtT<int>;

__host__ __device__ inline int sgn(int v) { return (v > 0) - (v < 0); }
__host__ __device__ inline int sgn(int64_t v) { return (v > 0) - (v < 0); }
__host__ __device__ inline int sgn(double v) { return (v > 0) - (v < 0); }

// Sklansky's coordinate differences and convexity: int with an int64 cross product, or float with a double one
__host__ __device__ inline int hull_sub(int a, int b) { return a - b; }
__host__ __device__ inline float hull_sub(float a, float b) { return fsub(a, b); }
__host__ __device__ inline int64_t hull_cross(int ay, int bx, int ax, int by) { return (int64_t)ay * bx - (int64_t)ax * by; }
__host__ __device__ inline double hull_cross(float ay, float bx, float ax, float by) {
    return dsub(dmul((double)ay, (double)bx), dmul((double)ax, (double)by));
}

template <class T>
__host__ __device__ inline bool pt_less(const PtT<T> *p, int a, int b) {
    return p[a].x < p[b].x || (p[a].x == p[b].x && p[a].y < p[b].y);
}

// std::sort as libstdc++ implements it (median-of-three quicksort down to runs of 16, heap sort past 2 log2(n) levels, then one
// insertion sort) of the indices idx[0..n) by (x, y), the order cv::convexHull sorts its point pointers in.  The comparison
// does not separate equal points; which of them cv2 ends up reporting is not always this sort's choice (see convex_hull).
template <class T>
__host__ __device__ inline void sift_down(const PtT<T> *p, int *a, int hole, int len, int value) {
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (pt_less(p, a[child], a[child - 1])) child--;
        a[hole] = a[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        a[hole] = a[child - 1];
        hole = child - 1;
    }
    int parent = (hole - 1) / 2;
    while (hole > top && pt_less(p, a[parent], value)) {
        a[hole] = a[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    a[hole] = value;
}

template <class T>
__host__ __device__ inline void heap_sort(const PtT<T> *p, int *a, int len) {
    if (len < 2) return;
    for (int parent = (len - 2) / 2;; --parent) {
        sift_down(p, a, parent, len, a[parent]);
        if (parent == 0) break;
    }
    for (int last = len - 1; last > 0; --last) {
        const int v = a[last];
        a[last] = a[0];
        sift_down(p, a, 0, last, v);
    }
}

__host__ __device__ inline void swap_idx(int *a, int i, int j) { const int t = a[i]; a[i] = a[j]; a[j] = t; }

template <class T>
__host__ __device__ inline void sort_points(const PtT<T> *p, int *a, int n) {
    if (n < 2) return;
    int lg = 0;
    while ((2 << lg) <= n) ++lg;
    // the recursion on the right part is made iterative with an explicit stack of (first, last, depth)
    int st[3 * 64], sp = 0;
    st[sp++] = 0; st[sp++] = n; st[sp++] = 2 * lg;
    while (sp) {
        int depth = st[--sp], last = st[--sp], first = st[--sp];
        while (last - first > 16) {
            if (depth == 0) {
                heap_sort(p, a + first, last - first);
                break;
            }
            --depth;
            const int mid = first + (last - first) / 2, x = first + 1, y = mid, z = last - 1;
            if (pt_less(p, a[x], a[y])) {
                if (pt_less(p, a[y], a[z])) swap_idx(a, first, y);
                else if (pt_less(p, a[x], a[z])) swap_idx(a, first, z);
                else swap_idx(a, first, x);
            } else if (pt_less(p, a[x], a[z])) swap_idx(a, first, x);
            else if (pt_less(p, a[y], a[z])) swap_idx(a, first, z);
            else swap_idx(a, first, y);
            int lo = first + 1, hi = last;
            for (;;) {
                while (pt_less(p, a[lo], a[first])) ++lo;
                --hi;
                while (pt_less(p, a[first], a[hi])) --hi;
                if (!(lo < hi)) break;
                swap_idx(a, lo, hi);
                ++lo;
            }
            // libstdc++ recurses into [cut, last) first, then continues with [first, cut); the order of the two parts does
            // not matter (they are disjoint), so the right part is pushed and the left one continues here
            st[sp++] = lo; st[sp++] = last; st[sp++] = depth;
            last = lo;
        }
    }
    auto linear_insert = [&](int i) {
        const int v = a[i];
        int j = i - 1;
        while (pt_less(p, v, a[j])) { a[j + 1] = a[j]; --j; }
        a[j + 1] = v;
    };
    const int head = n > 16 ? 16 : n;
    for (int i = 1; i < head; ++i) {
        if (pt_less(p, a[i], a[0])) {
            const int v = a[i];
            for (int j = i; j > 0; --j) a[j] = a[j - 1];
            a[0] = v;
        } else {
            linear_insert(i);
        }
    }
    for (int i = head; i < n; ++i) linear_insert(i);
}

// one monotone chain of cv::convexHull's Sklansky scan over the sorted order
template <class T>
__host__ __device__ inline int sklansky(const PtT<T> *p, const int *o, int start, int end, int *stack, int nsign, int sign2) {
    const int incr = end > start ? 1 : -1;
    int pprev = start, pcur = pprev + incr, pnext = pcur + incr;
    int stacksize = 3;
    if (start == end || (p[o[start]].x == p[o[end]].x && p[o[start]].y == p[o[end]].y)) {
        stack[0] = start;
        return 1;
    }
    stack[0] = pprev;
    stack[1] = pcur;
    stack[2] = pnext;
    end += incr;
    while (pnext != end) {
        const T cury = p[o[pcur]].y, nexty = p[o[pnext]].y, by = hull_sub(nexty, cury);
        if (sgn(by) != nsign) {
            const T ax = hull_sub(p[o[pcur]].x, p[o[pprev]].x), bx = hull_sub(p[o[pnext]].x, p[o[pcur]].x);
            const T ay = hull_sub(cury, p[o[pprev]].y);
            if (sgn(hull_cross(ay, bx, ax, by)) == sign2 && (ax != 0 || ay != 0)) {
                pprev = pcur;
                pcur = pnext;
                pnext += incr;
                stack[stacksize] = pnext;
                stacksize++;
            } else if (pprev == start) {
                pcur = pnext;
                stack[1] = pcur;
                pnext += incr;
                stack[2] = pnext;
            } else {
                stack[stacksize - 2] = pnext;
                pcur = pprev;
                pprev = stack[stacksize - 4];
                stacksize--;
            }
        } else {
            pnext += incr;
            stack[stacksize - 1] = pnext;
        }
    }
    return --stacksize;
}

// cv::convexHull(points, hull, clockwise = false): indices of the hull vertices into p[0..n) -- the vertices, orientation and
// cyclic order are cv2's; where a vertex occurs more than once in p, cv2 may report another of its copies and therefore start
// the (index-ordered) hull elsewhere (~0.5 % of contours, tests/test_db_boxes_cpu.py).  Scratch: o[n], stack[n + 2].  Returns the
// number of hull vertices.
template <class T>
__host__ __device__ inline int convex_hull(const PtT<T> *p, int n, int *o, int *stack, int *hull) {
    for (int i = 0; i < n; ++i) o[i] = i;
    sort_points(p, o, n);
    int miny = 0, maxy = 0;
    for (int i = 1; i < n; ++i) {
        const T y = p[o[i]].y;
        if (p[o[miny]].y > y) miny = i;
        if (p[o[maxy]].y < y) maxy = i;
    }
    int nout = 0;
    if (p[o[0]].x == p[o[n - 1]].x && p[o[0]].y == p[o[n - 1]].y) {
        hull[nout++] = o[0];
        return nout;
    }
    int *tl = stack;
    int tl_count = sklansky(p, o, 0, maxy, tl, -1, 1);
    int *tr = stack + tl_count;
    int tr_count = sklansky(p, o, n - 1, maxy, tr, -1, -1);
    {   // counter-clockwise: the two upper chains swap
        int *t = tl; tl = tr; tr = t;
        const int c = tl_count; tl_count = tr_count; tr_count = c;
    }
    for (int i = 0; i < tl_count - 1; ++i) hull[nout++] = o[tl[i]];
    for (int i = tr_count - 1; i > 0; --i) hull[nout++] = o[tr[i]];
    const int stop_idx = tr_count > 2 ? tr[1] : tl_count > 2 ? tl[tl_count - 2] : -1;
    int *bl = stack;
    int bl_count = sklansky(p, o, 0, miny, bl, 1, -1);
    int *br = stack + bl_count;
    int br_count = sklansky(p, o, n - 1, miny, br, 1, 1);
    if (stop_idx >= 0) {
        const int check_idx = bl_count > 2 ? bl[1] : bl_count + br_count > 2 ? br[2 - bl_count] : -1;
        if (check_idx == stop_idx ||
            (check_idx >= 0 && p[o[check_idx]].x == p[o[stop_idx]].x && p[o[check_idx]].y == p[o[stop_idx]].y)) {
            bl_count = bl_count < 2 ? bl_count : 2;          // all points on one line: the lower chain mirrors the upper one
            br_count = br_count < 2 ? br_count : 2;
        }
    }
    for (int i = 0; i < bl_count - 1; ++i) hull[nout++] = o[bl[i]];
    for (int i = br_count - 1; i > 0; --i) hull[nout++] = o[br[i]];
    // cyclic shift that makes the indices one ascending or descending run, if one exists
    if (nout >= 3) {
        int min_idx = 0, max_idx = 0, lt = 0;
        for (int i = 1; i < nout; ++i) {
            const int idx = hull[i];
            lt += hull[i - 1] < idx;
            if (lt > 1 && lt <= i - 2) break;
            if (idx < hull[min_idx]) min_idx = i;
            if (idx > hull[max_idx]) max_idx = i;
        }
        const int mmdist = min_idx > max_idx ? min_idx - max_idx : max_idx - min_idx;
        if ((mmdist == 1 || mmdist == nout - 1) && (lt <= 1 || lt >= nout - 2)) {
            const bool ascending = (max_idx + 1) % nout == min_idx;
            const int i0 = ascending ? min_idx : max_idx;
            if (i0 > 0) {
                int j = i0, i;
                for (i = 0; i < nout; ++i) {
                    const int curr = stack[i] = hull[j];
                    const int next_j = j + 1 < nout ? j + 1 : 0;
                    if (i < nout - 1 && (ascending != (curr < hull[next_j]))) break;
                    j = next_j;
                }
                if (i == nout)
                    for (int k = 0; k < nout; ++k) hull[k] = stack[k];
            }
        }
    }
    return nout;
}

}  // namespace mr_dbbox

namespace mr_dbbox {

struct Rect { float cx, cy, w, h, angle; };

__host__ __device__ inline float degrees(double rad) { return (float)(dmul(rad, 180.) / 3.14159265358979323846); }

// cv::minAreaRect of the hull points q[0..n) (float, in hull order): rotating calipers over the hull edges, the last
// rectangle of least area wins.  Scratch: vect[n] (edge vectors), inv[n] (1 / edge length).
__host__ __device__ inline Rect min_area_rect_hull(const float *qx, const float *qy, int n, float *vx, float *vy, float *inv) {
    Rect r{0.f, 0.f, 0.f, 0.f, 0.f};
    if (n > 2) {
        int left = 0, bottom = 0, right = 0, top = 0;
        float left_x = qx[0], right_x = qx[0], top_y = qy[0], bottom_y = qy[0];
        float px0 = qx[0], py0 = qy[0];
        for (int i = 0; i < n; ++i) {
            if (px0 < left_x) { left_x = px0; left = i; }
            if (px0 > right_x) { right_x = px0; right = i; }
            if (py0 > top_y) { top_y = py0; top = i; }
            if (py0 < bottom_y) { bottom_y = py0; bottom = i; }
            const int j = i + 1 < n ? i + 1 : 0;
            // float differences (exact for the integer points of contours), then double as cv2 has them
            const double dx = fsub(qx[j], px0), dy = fsub(qy[j], py0);
            vx[i] = (float)dx;
            vy[i] = (float)dy;
            inv[i] = (float)(1. / sqrt(dadd(dmul(dx, dx), dmul(dy, dy))));
            px0 = qx[j];
            py0 = qy[j];
        }
        float orientation = 0.f;
        {
            double ax = vx[n - 1], ay = vy[n - 1];
            for (int i = 0; i < n; ++i) {
                const double bx = vx[i], by = vy[i];
                const double convexity = dsub(dmul(ax, by), dmul(ay, bx));
                if (convexity != 0) {
                    orientation = convexity > 0 ? 1.f : -1.f;
                    break;
                }
                ax = bx;
                ay = by;
            }
        }
        float base_a = orientation, base_b = 0.f;
        int seq[4] = {bottom, right, top, left};
        float minarea = 3.402823466e+38f;
        int b_left = 0, b_bottom = 0;
        float b_a = 0.f, b_b = 0.f, b_w = 0.f, b_h = 0.f;
        for (int k = 0; k < n; ++k) {
            const float dp[4] = {
                fadd(fmul(base_a, vx[seq[0]]), fmul(base_b, vy[seq[0]])),
                fadd(fmul(-base_b, vx[seq[1]]), fmul(base_a, vy[seq[1]])),
                fsub(fmul(-base_a, vx[seq[2]]), fmul(base_b, vy[seq[2]])),
                fsub(fmul(base_b, vx[seq[3]]), fmul(base_a, vy[seq[3]])),
            };
            float maxcos = fmul(dp[0], inv[seq[0]]);
            int main_element = 0;
            for (int i = 1; i < 4; ++i) {
                const float c = fmul(dp[i], inv[seq[i]]);
                if (c > maxcos) { main_element = i; maxcos = c; }
            }
            const int pi = seq[main_element];
            const float lead_x = fmul(vx[pi], inv[pi]), lead_y = fmul(vy[pi], inv[pi]);
            switch (main_element) {
                case 0: base_a = lead_x; base_b = lead_y; break;
                case 1: base_a = lead_y; base_b = -lead_x; break;
                case 2: base_a = -lead_x; base_b = -lead_y; break;
                default: base_a = -lead_y; base_b = lead_x; break;
            }
            seq[main_element] += 1;
            if (seq[main_element] == n) seq[main_element] = 0;
            float dx = fsub(qx[seq[1]], qx[seq[3]]), dy = fsub(qy[seq[1]], qy[seq[3]]);
            const float width = fadd(fmul(dx, base_a), fmul(dy, base_b));
            dx = fsub(qx[seq[2]], qx[seq[0]]);
            dy = fsub(qy[seq[2]], qy[seq[0]]);
            const float height = fadd(fmul(-dx, base_b), fmul(dy, base_a));
            const float area = fmul(width, height);
            if (area <= minarea) {
                minarea = area;
                b_left = seq[3]; b_a = base_a; b_w = width; b_b = base_b; b_h = height; b_bottom = seq[0];
            }
        }
        const float A1 = b_a, B1 = b_b, A2 = -b_b, B2 = b_a;
        const float C1 = fadd(fmul(A1, qx[b_left]), fmul(qy[b_left], B1));
        const float C2 = fadd(fmul(A2, qx[b_bottom]), fmul(qy[b_bottom], B2));
        const float idet = 1.f / fsub(fmul(A1, B2), fmul(A2, B1));
        const float px = fmul(fsub(fmul(C1, B2), fmul(C2, B1)), idet);
        const float py = fmul(fsub(fmul(A1, C2), fmul(A2, C1)), idet);
        const float o1x = fmul(A1, b_w), o1y = fmul(B1, b_w), o2x = fmul(A2, b_h), o2y = fmul(B2, b_h);
        r.cx = fadd(px, fmul(fadd(o1x, o2x), 0.5f));
        r.cy = fadd(py, fmul(fadd(o1y, o2y), 0.5f));
        // degrees of the first side brought into [-90, 0) in double: a half turn keeps width and height, a quarter turn swaps them
        float w = (float)sqrt(dadd(dmul((double)o1x, (double)o1x), dmul((double)o1y, (double)o1y)));
        float h = (float)sqrt(dadd(dmul((double)o2x, (double)o2x), dmul((double)o2y, (double)o2y)));
        double deg = dmul(atan2((double)o1y, (double)o1x), 180.) / 3.14159265358979323846;
        if (deg >= 90.) deg = dsub(deg, 180.);
        else if (deg < -90.) deg = dadd(deg, 180.);
        if (deg >= 0.) {
            deg = dsub(deg, 90.);
            const float t = w; w = h; h = t;
        }
        r.w = w;
        r.h = h;
        r.angle = (float)deg;
        return r;
    } else if (n == 2) {
        r.cx = fmul(fadd(qx[0], qx[1]), 0.5f);
        r.cy = fmul(fadd(qy[0], qy[1]), 0.5f);
        const double dx = dsub((double)qx[1], (double)qx[0]), dy = dsub((double)qy[1], (double)qy[0]);
        r.w = (float)sqrt(dadd(dmul(dx, dx), dmul(dy, dy)));
        r.h = 0.f;
        r.angle = (float)atan2(dy, dx);
    } else if (n == 1) {
        r.cx = qx[0];
        r.cy = qy[0];
    }
    // degrees, brought into [-90, 0): a half turn keeps width and height, a quarter turn swaps them
    r.angle = degrees((double)r.angle);
    if (r.angle >= 90.f) r.angle = fsub(r.angle, 180.f);
    else if (r.angle < -90.f) r.angle = fadd(r.angle, 180.f);
    if (r.angle >= 0.f) {
        r.angle = fsub(r.angle, 90.f);
        const float t = r.w; r.w = r.h; r.h = t;
    }
    return r;
}

}  // namespace mr_dbbox

namespace mr_dbbox {

// cv2.boxPoints(rect): px[4], py[4]
__host__ __device__ inline void box_points(const Rect &r, float *px, float *py) {
    const double ang = (double)r.angle * 3.14159265358979323846 / 180.;
    const float b = fmul((float)cos(ang), 0.5f), a = fmul((float)sin(ang), 0.5f);
    px[0] = fsub(fsub(r.cx, fmul(a, r.h)), fmul(b, r.w));
    py[0] = fsub(fadd(r.cy, fmul(b, r.h)), fmul(a, r.w));
    px[1] = fsub(fadd(r.cx, fmul(a, r.h)), fmul(b, r.w));
    py[1] = fsub(fsub(r.cy, fmul(b, r.h)), fmul(a, r.w));
    px[2] = fsub(fmul(2.f, r.cx), px[0]);
    py[2] = fsub(fmul(2.f, r.cy), py[0]);
    px[3] = fsub(fmul(2.f, r.cx), px[1]);
    py[3] = fsub(fmul(2.f, r.cy), py[1]);
}

// cv2.boxPoints(rect) followed by get_mini_boxes' ordering (seg_detector_representer.py:125-145): the corners sorted by x
// (a stable sort), then of the two left ones the lower-y first, of the two right ones the lower-y second.  box[8] = (x, y) x 4.
// Returns min(width, height) ("sside").
__host__ __device__ inline float mini_box(const Rect &r, float *box) {
    float px[4], py[4];
    box_points(r, px, py);
    int o[4] = {0, 1, 2, 3};
    for (int i = 1; i < 4; ++i)                       // stable insertion sort by x
        for (int j = i; j > 0 && px[o[j]] < px[o[j - 1]]; --j) { const int t = o[j]; o[j] = o[j - 1]; o[j - 1] = t; }
    const bool l = py[o[1]] > py[o[0]], rgt = py[o[3]] > py[o[2]];
    const int sel[4] = {l ? o[0] : o[1], rgt ? o[2] : o[3], rgt ? o[3] : o[2], l ? o[1] : o[0]};
    for (int i = 0; i < 4; ++i) {
        box[2 * i] = px[sel[i]];
        box[2 * i + 1] = py[sel[i]];
    }
    return r.h < r.w ? r.h : r.w;
}

}  // namespace mr_dbbox

// ---- box_score_fast (seg_detector_representer.py:156-168): cv2.fillPoly of the box on a mask over its bounding rows and
// columns, then cv2.mean of the score map under the mask ----
namespace mr_dbbox {

struct L2 { int64_t x, y; };

// cv::clipLine on a width x height image (int64 endpoints, double intersections truncated toward zero)
__host__ __device__ inline bool clip_line(int64_t width, int64_t height, L2 &p1, L2 &p2) {
    const int64_t right = width - 1, bottom = height - 1;
    if (width <= 0 || height <= 0) return false;
    int64_t &x1 = p1.x, &y1 = p1.y, &x2 = p2.x, &y2 = p2.y;
    int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
    int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        int64_t a;
        if (c1 & 12) {
            a = c1 < 8 ? 0 : bottom;
            x1 += (int64_t)(dmul((double)(a - y1), (double)(x2 - x1)) / (double)(y2 - y1));
            y1 = a;
            c1 = (x1 < 0) + (x1 > right) * 2;
        }
        if (c2 & 12) {
            a = c2 < 8 ? 0 : bottom;
            x2 += (int64_t)(dmul((double)(a - y2), (double)(x2 - x1)) / (double)(y2 - y1));
            y2 = a;
            c2 = (x2 < 0) + (x2 > right) * 2;
        }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) {
                a = c1 == 1 ? 0 : right;
                y1 += (int64_t)(dmul((double)(a - x1), (double)(y2 - y1)) / (double)(x2 - x1));
                x1 = a;
                c1 = 0;
            }
            if (c2) {
                a = c2 == 1 ? 0 : right;
                y2 += (int64_t)(dmul((double)(a - x2), (double)(y2 - y1)) / (double)(x2 - x1));
                x2 = a;
                c2 = 0;
            }
        }
    }
    return (c1 | c2) == 0;
}

// One edge of cv::CollectPolyEdges (LINE_8, shift 0) from (x0, y0) to (x1, y1) on a width x height image: the ends of the
// 8-connected line cv2 draws for it, clipped to the image (*draw false when nothing of it is inside), and its PolyEdge of the
// scan-line fill in 16.16 fixed point (false for a horizontal edge, which has none).  An edge with an end outside the image
// takes the clipped ends' x (and their y unless the clipped segment is horizontal).
struct PolyEdge { int y0, y1; int64_t x, dx; int next; };

__host__ __device__ inline bool poly_edge(int x0, int y0, int x1, int y1, int width, int height, L2 &a, L2 &b, bool &draw,
                                          PolyEdge &ed) {
    const int XY_SHIFT = 16;
    const L2 pt0{(int64_t)x0 << XY_SHIFT, y0}, pt1{(int64_t)x1 << XY_SHIFT, y1};
    a = L2{x0, y0};
    b = L2{x1, y1};
    const bool outside = (uint64_t)a.x >= (uint64_t)width || (uint64_t)b.x >= (uint64_t)width ||
                         (uint64_t)a.y >= (uint64_t)height || (uint64_t)b.y >= (uint64_t)height;
    draw = !outside || clip_line(width, height, a, b);
    L2 c0 = pt0, c1 = pt1;
    if (outside) {
        if (a.y != b.y) { c0.y = a.y; c1.y = b.y; }
        c0.x = a.x << XY_SHIFT;
        c1.x = b.x << XY_SHIFT;
    }
    if (pt0.y == pt1.y) return false;
    ed.dx = (c1.x - c0.x) / (c1.y - c0.y);
    if (pt0.y < pt1.y) {
        ed.y0 = (int)pt0.y; ed.y1 = (int)pt1.y;
        ed.x = c0.x + (ed.y0 - c0.y) * ed.dx;
    } else {
        ed.y0 = (int)pt1.y; ed.y1 = (int)pt0.y;
        ed.x = c1.x + (ed.y0 - c1.y) * ed.dx;
    }
    return true;
}

// Line(img, a, b): cv::LineIterator(.., 8, leftToRight = true) over the clipped ends; visit(x, y) per pixel
template <class Visit>
__host__ __device__ inline void draw_line(L2 u, L2 v, Visit visit) {
    int64_t sy = 1, dx = v.x - u.x, dy = v.y - u.y;
    if (dx < 0) { dx = -dx; dy = -dy; const L2 t = u; u = v; v = t; }
    if (dy < 0) { dy = -dy; sy = -1; }
    const bool vert = dy > dx;
    if (vert) { const int64_t t = dx; dx = dy; dy = t; }
    int64_t err = dx - (dy + dy), x = u.x, y = u.y;
    for (int64_t k = 0; k <= dx; ++k) {
        visit((int)x, (int)y);
        const bool m = err < 0;
        err += -(dy + dy) + (m ? dx + dx : 0);
        if (vert) { y += sy; if (m) x += 1; }
        else { x += 1; if (m) y += sy; }
    }
}

// The pixels cv2.fillPoly(mask, [quad], 1) sets on a width x height mask (LINE_8, shift 0): the four edges drawn as
// 8-connected lines (clipped to the mask), and the scan-line fill of the edge collection in 16.16 fixed point (from the
// ceiling of the left edge to the floor of the right one, clipped to the mask).  visit(x, y) is called for every set pixel,
// possibly more than once; the scan-line fill stops before row y_stop (rows above it do not depend on the rows below).
template <class Visit>
__host__ __device__ inline void fill_quad(const int *q, int width, int height, int y_stop, Visit visit) {
    const int XY_SHIFT = 16;
    const int64_t XY_ONE = (int64_t)1 << XY_SHIFT;
    PolyEdge all[6];
    int ne = 0;
    for (int i = 0; i < 4; ++i) {
        const int k = (i + 3) & 3;
        L2 a, b;
        bool draw;
        if (poly_edge(q[2 * k], q[2 * k + 1], q[2 * i], q[2 * i + 1], width, height, a, b, draw, all[ne])) ++ne;
        if (draw) draw_line(a, b, visit);
    }
    // FillEdgeCollection
    if (ne < 2) return;
    int y_max = INT32_MIN, y_min = INT32_MAX;
    int64_t x_max = -1, x_min = INT64_MAX;
    for (int i = 0; i < ne; ++i) {
        const int64_t x1 = all[i].x + (int64_t)(all[i].y1 - all[i].y0) * all[i].dx;
        y_min = all[i].y0 < y_min ? all[i].y0 : y_min;
        y_max = all[i].y1 > y_max ? all[i].y1 : y_max;
        x_min = all[i].x < x_min ? all[i].x : x_min;
        x_max = all[i].x > x_max ? all[i].x : x_max;
        x_min = x1 < x_min ? x1 : x_min;
        x_max = x1 > x_max ? x1 : x_max;
    }
    if (y_max < 0 || y_min >= height || x_max < 0 || x_min >= ((int64_t)width << XY_SHIFT)) return;
    for (int i = 1; i < ne; ++i)                 // std::sort of <= 4 edges (an insertion sort) by (y0, x, dx)
        for (int j = i; j > 0; --j) {
            const PolyEdge &p = all[j - 1], &c = all[j];
            if (!(c.y0 != p.y0 ? c.y0 < p.y0 : c.x != p.x ? c.x < p.x : c.dx < p.dx)) break;
            const PolyEdge t = all[j]; all[j] = all[j - 1]; all[j - 1] = t;
        }
    const int TMP = 5;                           // the list head; edge `ne` is the y0 = INT_MAX sentinel
    all[ne].y0 = INT32_MAX;
    all[TMP].next = -1;
    int i = 0;
    y_max = y_max < height ? y_max : height;
    y_max = y_max < y_stop ? y_max : y_stop;
    for (int y = all[0].y0; y < y_max; y++) {
        int prelast = TMP, last = all[TMP].next, keep_prelast, draw = 0;
        while (last >= 0 || all[i].y0 == y) {
            if (last >= 0 && all[last].y1 == y) {    // the edge ends here
                all[prelast].next = all[last].next;
                last = all[last].next;
                continue;
            }
            keep_prelast = prelast;
            if (last >= 0 && (all[i].y0 > y || all[last].x < all[i].x)) {
                prelast = last;
                last = all[last].next;
            } else if (i < ne) {                     // the next edge starts here
                all[prelast].next = i;
                all[i].next = last;
                prelast = i;
                ++i;
            } else {
                break;
            }
            if (draw) {
                if (y >= 0) {
                    const int64_t xa = all[keep_prelast].x, xb = all[prelast].x;
                    int x1 = (int)(((xa > xb ? xb : xa) + XY_ONE - 1) >> XY_SHIFT), x2 = (int)((xa > xb ? xa : xb) >> XY_SHIFT);
                    if (x1 < width && x2 >= 0) {
                        if (x1 < 0) x1 = 0;
                        if (x2 >= width) x2 = width - 1;
                        for (int x = x1; x <= x2; ++x) visit(x, y);
                    }
                }
                all[keep_prelast].x += all[keep_prelast].dx;
                all[prelast].x += all[prelast].dx;
            }
            draw ^= 1;
        }
        keep_prelast = -1;                       // bubble sort of the active list by x
        do {
            prelast = TMP;
            last = all[TMP].next;
            int last_exchange = -1;
            while (last != keep_prelast && last >= 0 && all[last].next >= 0) {
                const int te = all[last].next;
                if (all[last].x > all[te].x) {
                    all[prelast].next = te;
                    all[last].next = all[te].next;
                    all[te].next = last;
                    prelast = te;
                    last_exchange = prelast;
                } else {
                    prelast = last;
                    last = te;
                }
            }
            if (last_exchange < 0) break;
            keep_prelast = last_exchange;
        } while (keep_prelast != all[TMP].next && keep_prelast != TMP);
    }
}

}  // namespace mr_dbbox

namespace mr_dbbox {

// box_score_fast(pred, box): pred is H x W (row stride W), box[8] the float corners.  The mask covers the box's bounding
// columns / rows clipped to the map (floor / ceil of the corner extremes); the corners are shifted by the mask's origin and
// truncated toward zero (astype(np.int32)); the score is cv2.mean: the masked values summed in double in raster order, times
// 1 / count.  The mask is built a band of rows at a time in 8192 bits, so no scratch memory is needed.
__host__ __device__ inline double box_score(const float *pred, int H, int W, const float *box) {
    float mnx = box[0], mxx = box[0], mny = box[1], mxy = box[1];
    for (int i = 1; i < 4; ++i) {
        mnx = box[2 * i] < mnx ? box[2 * i] : mnx;
        mxx = box[2 * i] > mxx ? box[2 * i] : mxx;
        mny = box[2 * i + 1] < mny ? box[2 * i + 1] : mny;
        mxy = box[2 * i + 1] > mxy ? box[2 * i + 1] : mxy;
    }
    auto clampi = [](float v, int hi) { const int64_t i = (int64_t)v; return (int)(i < 0 ? 0 : i > hi ? hi : i); };
    const int xmin = clampi(floorf(mnx), W - 1), xmax = clampi(ceilf(mxx), W - 1);
    const int ymin = clampi(floorf(mny), H - 1), ymax = clampi(ceilf(mxy), H - 1);
    int q[8];
    for (int i = 0; i < 4; ++i) {
        q[2 * i] = (int)(float)dsub((double)box[2 * i], (double)xmin);
        q[2 * i + 1] = (int)(float)dsub((double)box[2 * i + 1], (double)ymin);
    }
    const int bw = xmax - xmin + 1, bh = ymax - ymin + 1;
    // mask bits of a band of rows: as many whole rows as fit 8192 bits, or one row in 8192-column pieces, so that the values
    // are always summed in raster order
    constexpr int kWords = 256;
    const int wpr = (bw + 31) / 32 < kWords ? (bw + 31) / 32 : kWords, rows = kWords / wpr, cols = 32 * wpr;
    double s = 0.;
    int64_t nz = 0;
    uint32_t bits[kWords];
    for (int y0 = 0; y0 < bh; y0 += rows)
        for (int x0 = 0; x0 < bw; x0 += cols) {
            for (int k = 0; k < kWords; ++k) bits[k] = 0u;
            fill_quad(q, bw, bh, y0 + rows, [&](int x, int y) {
                if (y >= y0 && y < y0 + rows && x >= x0 && x < x0 + cols)
                    bits[(y - y0) * wpr + ((x - x0) >> 5)] |= 1u << ((x - x0) & 31);
            });
            for (int r = 0; r < rows && y0 + r < bh; ++r) {
                const float *row = pred + (int64_t)(ymin + y0 + r) * W + xmin + x0;
                for (int k = 0; k < wpr; ++k)
                    for (uint32_t b = bits[r * wpr + k]; b; b &= b - 1) {
                        int j = 0;
                        while (!((b >> j) & 1u)) ++j;
                        s = dadd(s, (double)row[32 * k + j]);
                        ++nz;
                    }
            }
        }
    return nz ? dmul(s, 1. / (double)nz) : 0.;
}

}  // namespace mr_dbbox

// ---- unclip (seg_detector_representer.py:97-123): distance = Polygon(box).area * 1.5 / Polygon(box).length (GEOS ring
// formulas in double), then pyclipper's PyclipperOffset().AddPath(box, JT_ROUND, ET_CLOSEDPOLYGON).Execute(distance), restated
// from the published Clipper 6.4.2 ClipperOffset (miter limit 2, arc tolerance 0.25): AddPath on the corners truncated to
// integers, FixOrientations, DoOffset with DoRound, Round() half away from zero.  The ctUnion / pftPositive clean-up that
// Execute runs last is not restated: for the offset of a box it yields the same region, whose convex hull -- all the second
// cv2.minAreaRect looks at -- is that of the offset path; only the order of its points, and with it the tie class of DESIGN §7,
// can differ.  This restatement is not pinned against pyclipper (not a dependency of the project); tests pin its invariants. ----
namespace mr_dbbox {

// GEOS Area::ofRing and Length::ofLine of the closed ring box[0..3], box[0] (float or double corners)
template <class T>
__host__ __device__ inline void ring_area_length(const T *box, double &area, double &length) {
    double x[5], y[5];
    for (int i = 0; i < 5; ++i) { x[i] = box[2 * (i & 3)]; y[i] = box[2 * (i & 3) + 1]; }
    double sum = 0., len = 0.;
    for (int i = 1; i < 4; ++i) sum = dadd(sum, dmul(dsub(x[i], x[0]), dsub(y[i - 1], y[i + 1])));
    for (int i = 0; i < 4; ++i) {
        const double dx = dsub(x[i + 1], x[i]), dy = dsub(y[i + 1], y[i]);
        len = dadd(len, sqrt(dadd(dmul(dx, dx), dmul(dy, dy))));
    }
    area = fabs(sum / 2.);
    length = len;
}

__host__ __device__ inline double unclip_distance(const float *box) {
    double area, len;
    ring_area_length(box, area, len);
    return dmul(area, 1.5) / len;
}

__host__ __device__ inline int64_t clipper_round(double v) { return v < 0 ? (int64_t)dsub(v, 0.5) : (int64_t)dadd(v, 0.5); }

// The raw offset path of the box (float or double corners; delta > 0 pads, delta < 0 shrinks) before Execute's clean-up:
// int points into ox / oy, at most cap of them.  Returns the number of points, 0 when the truncated box has fewer than three
// distinct points (Clipper then has no path), -1 when cap is too small.
template <class T>
__host__ __device__ inline int unclip_offset(const T *box, double delta, int *ox, int *oy, int cap) {
    // AddPath: truncation to cInt, trailing copies of the first point and consecutive duplicates dropped
    int64_t px[4], py[4];
    int hi = 3;
    for (int i = 0; i < 4; ++i) { px[i] = (int64_t)box[2 * i]; py[i] = (int64_t)box[2 * i + 1]; }
    while (hi > 0 && px[0] == px[hi] && py[0] == py[hi]) hi--;
    int64_t sx[4], sy[4];
    int len = 1;
    sx[0] = px[0]; sy[0] = py[0];
    for (int i = 1; i <= hi; ++i)
        if (sx[len - 1] != px[i] || sy[len - 1] != py[i]) { sx[len] = px[i]; sy[len] = py[i]; ++len; }
    if (len < 3) return 0;
    // FixOrientations: the (only) path is reversed unless Orientation(path), i.e. Area(path) >= 0
    double a = 0.;
    for (int i = 0, j = len - 1; i < len; j = i++)
        a = dadd(a, dmul(dadd((double)sx[j], (double)sx[i]), dsub((double)sy[j], (double)sy[i])));
    if (!(-a * 0.5 >= 0.))
        for (int i = 0; i < len / 2; ++i) {
            int64_t t = sx[i]; sx[i] = sx[len - 1 - i]; sx[len - 1 - i] = t;
            t = sy[i]; sy[i] = sy[len - 1 - i]; sy[len - 1 - i] = t;
        }
    // DoOffset
    const double PI = 3.141592653589793238, TWO_PI = PI * 2;
    const double y = 0.25 > fabs(delta) * 0.25 ? fabs(delta) * 0.25 : 0.25;
    double steps = PI / acos(1. - y / fabs(delta));
    if (steps > fabs(delta) * PI) steps = fabs(delta) * PI;
    double msin = sin(TWO_PI / steps);
    const double mcos = cos(TWO_PI / steps), steps_per_rad = steps / TWO_PI;
    if (delta < 0.) msin = -msin;
    double nx[4], ny[4];
    for (int j = 0; j < len; ++j) {                 // GetUnitNormal(p[j], p[j + 1 (mod len)])
        const int k = j + 1 < len ? j + 1 : 0;
        double dx = (double)(sx[k] - sx[j]), dy = (double)(sy[k] - sy[j]);
        const double f = 1. / sqrt(dadd(dmul(dx, dx), dmul(dy, dy)));
        dx = dmul(dx, f);
        dy = dmul(dy, f);
        nx[j] = dy;
        ny[j] = -dx;
    }
    int n = 0;
    auto push = [&](int64_t X, int64_t Y) {
        if (n < cap) { ox[n] = (int)X; oy[n] = (int)Y; }
        ++n;
    };
    for (int j = 0, k = len - 1; j < len; k = j, ++j) {   // OffsetPoint(j, k, jtRound)
        double sinA = dsub(dmul(nx[k], ny[j]), dmul(nx[j], ny[k]));
        if (fabs(dmul(sinA, delta)) < 1.0) {
            const double cosA = dadd(dmul(nx[k], nx[j]), dmul(ny[j], ny[k]));
            if (cosA > 0) {
                push(clipper_round(dadd((double)sx[j], dmul(nx[k], delta))), clipper_round(dadd((double)sy[j], dmul(ny[k], delta))));
                continue;
            }
        } else if (sinA > 1.0) {
            sinA = 1.0;
        } else if (sinA < -1.0) {
            sinA = -1.0;
        }
        if (dmul(sinA, delta) < 0) {
            push(clipper_round(dadd((double)sx[j], dmul(nx[k], delta))), clipper_round(dadd((double)sy[j], dmul(ny[k], delta))));
            push(sx[j], sy[j]);
            push(clipper_round(dadd((double)sx[j], dmul(nx[j], delta))), clipper_round(dadd((double)sy[j], dmul(ny[j], delta))));
        } else {                                    // DoRound
            const double ang = atan2(sinA, dadd(dmul(nx[k], nx[j]), dmul(ny[k], ny[j])));
            int st = (int)clipper_round(dmul(steps_per_rad, fabs(ang)));
            st = st > 1 ? st : 1;
            double X = nx[k], Y = ny[k];
            for (int i = 0; i < st; ++i) {
                push(clipper_round(dadd((double)sx[j], dmul(X, delta))), clipper_round(dadd((double)sy[j], dmul(Y, delta))));
                const double X2 = X;
                X = dsub(dmul(X, mcos), dmul(msin, Y));
                Y = dadd(dmul(X2, msin), dmul(Y, mcos));
            }
            push(clipper_round(dadd((double)sx[j], dmul(nx[j], delta))), clipper_round(dadd((double)sy[j], dmul(ny[j], delta))));
        }
    }
    return n <= cap ? n : -1;
}

// Points of the offset path for a box whose distance is delta, bounded for the scratch of the second box
__host__ __device__ inline int unclip_max_points(double delta) {
    const double PI = 3.141592653589793238;
    const double y = 0.25 > fabs(delta) * 0.25 ? fabs(delta) * 0.25 : 0.25;
    double steps = PI / acos(1. - y / fabs(delta));
    if (steps > fabs(delta) * PI) steps = fabs(delta) * PI;
    return (int)steps + 16;                          // one turn of round joins plus up to three points per corner
}

// box[:, k] = np.clip(np.round(box[:, k] / size * dest), 0, dest) in float32 with round-half-even (:107-110)
__host__ __device__ inline int rescale(float v, int size, int dest) {
#ifdef __CUDA_ARCH__
    float r = rintf(__fmul_rn(__fdiv_rn(v, (float)size), (float)dest));
#else
    float r = rintf(v / (float)size * (float)dest);
#endif
    r = r < 0.f ? 0.f : r > (float)dest ? (float)dest : r;
    return (int)r;
}

}  // namespace mr_dbbox
