// Geometry of the DB detector's validation measure (QuadMeasurer -> DetectionIoUEvaluator.evaluate_image,
// concern/icdar2015_eval/detection/iou.py:13-179) for 4-point rings, shared by the CUDA kernels (db_measure.cu) and by a
// host-side harness (tests/host_harness/db_measure_core_host.cpp) that runs the SAME routines on the CPU.  float64, every
// operation rounded on its own (no fused multiply-add), so host and device give the same bits.
//
// What is restated here, standing in for the shapely calls of the evaluator:
//   * Polygon(p).is_valid and .is_simple (GEOS IsValidOp on one ring): ring_valid.  The orientation and area signs it needs
//     are exact (products split with fma, summed as a floating-point expansion), not compared against a tolerance;
//   * Polygon(p).area: the GEOS ring formula (ring_area), bit-equal to Area::ofRing;
//   * Polygon(a).intersection(Polygon(b)).area: the rings split into at most two convex pieces each (ring_prepare), every
//     piece pair clipped by Sutherland-Hodgman (clip_area).  A crossing with a horizontal or vertical clip edge takes that
//     edge's coordinate exactly, so axis-aligned integer boxes give exact areas;
//   * Polygon(a).union(Polygon(b)).area as area(a) + area(b) - intersection (DESIGN §7).
// This is not pinned against shapely, which is not a dependency; oracle/db_measure_port.py restates it in exact rational
// arithmetic and the CPU tests compare the two.
#pragma once
#include <math.h>

#include "db_boxes_core.cuh"

namespace mr_dbmeas {

using mr_dbbox::dadd;
using mr_dbbox::dmul;
using mr_dbbox::dsub;

#ifdef __CUDA_ARCH__
__device__ __forceinline__ double dfma(double a, double b, double c) { return __fma_rn(a, b, c); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
#else
inline double dfma(double a, double b, double c) { return fma(a, b, c); }
inline double ddiv(double a, double b) { return a / b; }
#endif

// ---- exact signs ----

// Sign of the exact sum of the n products a[i] * b[i] (n <= 8): each product is split into its rounded value and its exact
// error, and the 2n terms are summed into a nonoverlapping expansion (Shewchuk's Grow-Expansion with zero elimination), whose
// largest component carries the sign of the sum.
__host__ __device__ inline int sign_of_products(const double *a, const double *b, int n) {
    double e[16];
    int m = 0;
    for (int i = 0; i < 2 * n; ++i) {
        const double p = dmul(a[i >> 1], b[i >> 1]);
        double q = (i & 1) ? dfma(a[i >> 1], b[i >> 1], -p) : p;
        int k = 0;
        for (int j = 0; j < m; ++j) {                 // TwoSum(q, e[j])
            const double s = dadd(q, e[j]);
            const double bv = dsub(s, q);
            const double err = dadd(dsub(q, dsub(s, bv)), dsub(e[j], bv));
            if (err != 0.) e[k++] = err;
            q = s;
        }
        if (q != 0.) e[k++] = q;
        m = k;
    }
    return m == 0 ? 0 : (e[m - 1] > 0. ? 1 : -1);
}

// exact sign of (b - a) x (c - a) = bx cy - bx ay - ax cy - by cx + by ax + ay cx
__host__ __device__ inline int orient(double ax, double ay, double bx, double by, double cx, double cy) {
    const double l[6] = {bx, -bx, -ax, -by, by, ay};
    const double r[6] = {cy, ay, cy, cx, ax, cx};
    return sign_of_products(l, r, 6);
}

// exact sign of twice the signed area (shoelace) of the n-point ring x, y (n <= 4)
__host__ __device__ inline int area_sign(const double *x, const double *y, int n) {
    double l[8], r[8];
    for (int i = 0; i < n; ++i) {
        const int j = i + 1 == n ? 0 : i + 1;
        l[2 * i] = x[i];  r[2 * i] = y[j];
        l[2 * i + 1] = -x[j]; r[2 * i + 1] = y[i];
    }
    return sign_of_products(l, r, 2 * n);
}

// p lies in the closed bounding box of segment a-b (with orient(a, b, p) == 0: p lies on the segment)
__host__ __device__ inline bool in_box(double ax, double ay, double bx, double by, double px, double py) {
    return fmin(ax, bx) <= px && px <= fmax(ax, bx) && fmin(ay, by) <= py && py <= fmax(ay, by);
}

// closed segments a-b and c-d share a point
__host__ __device__ inline bool segments_touch(double ax, double ay, double bx, double by, double cx, double cy, double dx,
                                               double dy) {
    const int o1 = orient(ax, ay, bx, by, cx, cy), o2 = orient(ax, ay, bx, by, dx, dy);
    const int o3 = orient(cx, cy, dx, dy, ax, ay), o4 = orient(cx, cy, dx, dy, bx, by);
    if (o1 * o2 < 0 && o3 * o4 < 0) return true;
    return (o1 == 0 && in_box(ax, ay, bx, by, cx, cy)) || (o2 == 0 && in_box(ax, ay, bx, by, dx, dy)) ||
           (o3 == 0 && in_box(cx, cy, dx, dy, ax, ay)) || (o4 == 0 && in_box(cx, cy, dx, dy, bx, by));
}

// ---- one ring ----

// The ring of a [4, 2] polygon, prepared for the measure: validity, GEOS area, bounding box and convex pieces (each
// counter-clockwise, 3 or 4 vertices).
struct Ring {
    double px[2][4], py[2][4];  // convex pieces
    double box[4];              // xmin, ymin, xmax, ymax
    double area;
    int np[2];                  // vertices of each piece
    int pieces;                 // 0 (invalid ring), 1 or 2
    int valid;
};

// GEOS Area::ofRing of the closed 4-point ring
__host__ __device__ inline double ring_area(const double *q) {
    double s = 0.;
    const double x0 = q[0];
    for (int i = 1; i < 4; ++i) {
        const double xi = q[2 * i], ya = q[2 * (i - 1) + 1], yb = q[2 * ((i + 1) & 3) + 1];
        s = dadd(s, dmul(dsub(xi, x0), dsub(ya, yb)));
    }
    return fabs(s / 2.0);
}

// Polygon(q).is_valid and Polygon(q).is_simple for the [4, 2] ring q: every coordinate finite; at least 3 distinct vertices
// once consecutive duplicates are dropped (cyclically); no two non-adjacent edges share a point; no two adjacent edges
// overlap beyond their shared vertex; nonzero area.  On success x, y hold the m distinct vertices.
__host__ __device__ inline bool ring_valid(const double *q, double *x, double *y, int *m_out) {
    for (int k = 0; k < 8; ++k)
        if (!isfinite(q[k])) return false;
    int m = 0;
    for (int i = 0; i < 4; ++i) {
        const double vx = q[2 * i], vy = q[2 * i + 1];
        if (m > 0 && vx == x[m - 1] && vy == y[m - 1]) continue;
        x[m] = vx; y[m] = vy; ++m;
    }
    while (m > 1 && x[m - 1] == x[0] && y[m - 1] == y[0]) --m;
    *m_out = m;
    if (m < 3) return false;
    for (int i = 0; i < m; ++i) {                      // adjacent edges (a, b), (b, c): no fold-back at b
        const int a = (i + m - 1) % m, c = (i + 1) % m;
        if (orient(x[a], y[a], x[i], y[i], x[c], y[c]) != 0) continue;
        // collinear: the edges overlap iff a and c lie on the same side of b along the line
        const bool fold = x[a] != x[i] ? ((x[a] > x[i]) == (x[c] > x[i])) : ((y[a] > y[i]) == (y[c] > y[i]));
        if (fold) return false;
    }
    if (m == 4)
        for (int i = 0; i < 2; ++i)                     // edges (0,1)-(2,3) and (1,2)-(3,0)
            if (segments_touch(x[i], y[i], x[i + 1], y[i + 1], x[i + 2], y[i + 2], x[(i + 3) & 3], y[(i + 3) & 3])) return false;
    return area_sign(x, y, m) != 0;
}

// validity, area, bounding box and convex pieces of the [4, 2] ring q
__host__ __device__ inline Ring ring_prepare(const double *q) {
    Ring r;
    double x[4], y[4];
    int m = 0;
    r.pieces = 0;
    r.np[0] = r.np[1] = 0;
    r.valid = ring_valid(q, x, y, &m);
    r.area = r.valid ? ring_area(q) : 0.;
    r.box[0] = r.box[1] = r.box[2] = r.box[3] = 0.;
    if (!r.valid) return r;
    r.box[0] = r.box[2] = x[0];
    r.box[1] = r.box[3] = y[0];
    for (int i = 1; i < m; ++i) {
        r.box[0] = fmin(r.box[0], x[i]); r.box[2] = fmax(r.box[2], x[i]);
        r.box[1] = fmin(r.box[1], y[i]); r.box[3] = fmax(r.box[3], y[i]);
    }
    const int s = area_sign(x, y, m);
    int reflex = -1;                                    // a simple quad has at most one reflex vertex
    for (int i = 0; i < m && m == 4; ++i)
        if (orient(x[(i + 3) & 3], y[(i + 3) & 3], x[i], y[i], x[(i + 1) & 3], y[(i + 1) & 3]) == -s) reflex = i;
    auto put = [&](int p, int a, int b, int c, int d, int n) {     // vertices a, b, c (, d) counter-clockwise
        const int v[4] = {a, b, c, d};
        for (int k = 0; k < n; ++k) {
            const int src = s > 0 ? v[k] : v[n - 1 - k];
            r.px[p][k] = x[src]; r.py[p][k] = y[src];
        }
        r.np[p] = n;
    };
    if (reflex < 0) {
        put(0, 0, 1, 2, 3, m);
        r.pieces = 1;
    } else {                                            // cut along the diagonal from the reflex vertex
        const int a = reflex;
        put(0, a, (a + 1) & 3, (a + 2) & 3, 0, 3);
        put(1, a, (a + 2) & 3, (a + 3) & 3, 0, 3);
        r.pieces = 2;
    }
    return r;
}

// ---- intersection ----

__host__ __device__ inline bool boxes_overlap(const double *a, const double *b) {
    return fmax(a[0], b[0]) < fmin(a[2], b[2]) && fmax(a[1], b[1]) < fmin(a[3], b[3]);
}

// Vertices a Sutherland-Hodgman pass can leave, whatever its inside tests decide.  A pass over c vertices of which k are
// inside emits the k and one crossing per inside/outside change; there are at most 2 min(k, c - k) changes around the
// ring, so it emits at most min(3k, 2c - k) <= 3c/2.  Four passes from at most 4 vertices: 4 -> 6 -> 9 -> 13 -> 19.  The
// bound does not assume the result is convex, so rounding in the tests cannot overflow the buffers.
constexpr int kClipMax = 19;

// Area of the intersection of two convex counter-clockwise polygons (n, m <= 4): the subject a clipped by every edge of
// the clip polygon b in turn (Sutherland-Hodgman), then the shoelace of what is left.
__host__ __device__ inline double clip_area(const double *ax, const double *ay, int n, const double *bx, const double *by, int m) {
    double ux[kClipMax], uy[kClipMax], vx[kClipMax], vy[kClipMax];
    int cnt = n;
    for (int i = 0; i < n; ++i) { ux[i] = ax[i]; uy[i] = ay[i]; }
    for (int e = 0; e < m && cnt > 0; ++e) {
        const double ex0 = bx[e], ey0 = by[e], ex1 = bx[(e + 1) % m], ey1 = by[(e + 1) % m];
        const double dx = dsub(ex1, ex0), dy = dsub(ey1, ey0);
        auto side = [&](double px, double py) { return dsub(dmul(dx, dsub(py, ey0)), dmul(dy, dsub(px, ex0))); };
        int out = 0;
        double sp = side(ux[cnt - 1], uy[cnt - 1]);
        double prx = ux[cnt - 1], pry = uy[cnt - 1];
        for (int i = 0; i < cnt; ++i) {
            const double cx = ux[i], cy = uy[i], sc = side(cx, cy);
            const bool pin = sp >= 0., cin = sc >= 0.;
            if (pin != cin) {                           // the edge prev -> cur crosses the clip line
                const double t = ddiv(sp, dsub(sp, sc));
                double ix = dadd(prx, dmul(t, dsub(cx, prx))), iy = dadd(pry, dmul(t, dsub(cy, pry)));
                if (dy == 0.) iy = ey0;                 // horizontal clip edge: its y exactly
                if (dx == 0.) ix = ex0;                 // vertical clip edge: its x exactly
                vx[out] = ix; vy[out] = iy; ++out;
            }
            if (cin) { vx[out] = cx; vy[out] = cy; ++out; }
            sp = sc; prx = cx; pry = cy;
        }
        cnt = out;
        for (int i = 0; i < cnt; ++i) { ux[i] = vx[i]; uy[i] = vy[i]; }
    }
    if (cnt < 3) return 0.;
    double s = 0.;                                      // fan from the first vertex, in coordinates relative to it
    for (int i = 1; i + 1 < cnt; ++i) {
        const double x1 = dsub(ux[i], ux[0]), y1 = dsub(uy[i], uy[0]), x2 = dsub(ux[i + 1], ux[0]), y2 = dsub(uy[i + 1], uy[0]);
        s = dadd(s, dsub(dmul(x1, y2), dmul(x2, y1)));
    }
    return s > 0. ? s / 2.0 : 0.;
}

// Polygon(a).intersection(Polygon(b)).area of two valid rings.  The ring of smaller area is the one clipped: a ring inside
// the other then comes out unchanged, without crossings computed against its edges (thin slivers keep their area).
__host__ __device__ inline double intersection_area(const Ring &ra, const Ring &rb) {
    if (!boxes_overlap(ra.box, rb.box)) return 0.;
    const bool swap = rb.area < ra.area;
    const Ring &a = swap ? rb : ra, &b = swap ? ra : rb;
    double s = 0.;
    for (int i = 0; i < a.pieces; ++i)
        for (int j = 0; j < b.pieces; ++j) {
            double pa[4] = {a.px[i][0], a.py[i][0], a.px[i][0], a.py[i][0]}, pb[4] = {b.px[j][0], b.py[j][0], b.px[j][0], b.py[j][0]};
            for (int k = 1; k < a.np[i]; ++k) {
                pa[0] = fmin(pa[0], a.px[i][k]); pa[2] = fmax(pa[2], a.px[i][k]);
                pa[1] = fmin(pa[1], a.py[i][k]); pa[3] = fmax(pa[3], a.py[i][k]);
            }
            for (int k = 1; k < b.np[j]; ++k) {
                pb[0] = fmin(pb[0], b.px[j][k]); pb[2] = fmax(pb[2], b.px[j][k]);
                pb[1] = fmin(pb[1], b.py[j][k]); pb[3] = fmax(pb[3], b.py[j][k]);
            }
            if (!boxes_overlap(pa, pb)) continue;
            s = dadd(s, clip_area(a.px[i], a.py[i], a.np[i], b.px[j], b.py[j], b.np[j]));
        }
    return s;
}

// get_intersection_over_union(det, gt) and the don't-care precision intersection / area(det) of two valid rings
__host__ __device__ inline void iou_precision(const Ring &gt, const Ring &det, double *iou, double *precision) {
    const double inter = intersection_area(gt, det);
    const double uni = dsub(dadd(det.area, gt.area), inter);
    *iou = uni > 0. ? ddiv(inter, uni) : 0.;
    *precision = det.area == 0. ? 0. : ddiv(inter, det.area);
}

// evaluate_image's per-image metrics, with its branches; hmean = 2.0 * p * r / (p + r) evaluated left to right
__host__ __device__ inline void image_metrics(int gt_care, int det_care, int matched, double *p, double *r, double *h) {
    if (gt_care == 0) {
        *r = 1.;
        *p = det_care > 0 ? 0. : 1.;
    } else {
        *r = ddiv((double)matched, (double)gt_care);
        *p = det_care == 0 ? 0. : ddiv((double)matched, (double)det_care);
    }
    const double sum = dadd(*p, *r);
    *h = sum == 0. ? 0. : ddiv(dmul(dmul(2.0, *p), *r), sum);
}

}  // namespace mr_dbmeas
