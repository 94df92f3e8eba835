// Per-polygon and per-pixel routines of the DB detector's training targets (data/processes/make_seg_detection_data.py:21-100,
// make_border_map.py:24-121), shared by the CUDA kernels (db_targets.cu) and by a host-side harness
// (tests/host_harness/db_targets_core_host.cpp) that runs the SAME routines on the CPU.  Builds on db_boxes_core.cuh: the
// round offset (unclip_offset), the GEOS ring formulas and cv2's line clipping.
//
// What is restated here:
//   * validate_polygons in the polygon's dtype (clip, the polygon_area sign test and the (0,3,2,1) reversal, |area| < 1);
//   * Clipper 6.4.2's ClipperOffset::Execute clean-up for the raw offset path of one quad (clean_offset), see below;
//   * cv2.fillPoly of one integer polygon, split so that every pixel is decided on its own (fill_edge, fill_bounds,
//     pixel_filled);
//   * MakeBorderMap.distance for one pixel and one edge, in float64 without fused multiply-add (edge_distance).
//
// The clean-up.  Execute unions the raw offset path with itself: ctUnion / pftPositive for a pad, and for a shrink the
// complement trick (outer rectangle, reversed, pftNegative, first polygon dropped), whose effect is the components of
// {winding >= 1}.  Both are therefore the boundary of {winding of the raw path >= 1}.  It is computed on the planar
// arrangement of the raw edges: every pair of raw edges that properly cross is split at the crossing, rounded as Clipper's
// IntersectPoint rounds it (see clipper_intersect), and an edge with a raw vertex inside it at that vertex; a piece of a raw edge is kept when the winding number just left of it is
// 1 (just right of it it is then 0); the kept pieces are chained into loops, at a node with several ways out taking the
// sharpest left turn; duplicate and collinear points are dropped (PreserveCollinear is false); and of several loops the one
// of largest |area| is the result (the first traced on ties), the others are counted.  pyclipper is not a dependency of
// the project, so this is not pinned against it; tests pin its invariants and an independent Python restatement
// (oracle/db_targets_port.py) follows the same rules.
#pragma once
#include "db_boxes_core.cuh"

namespace mr_dbtgt {

using mr_dbbox::clipper_round;
using mr_dbbox::dadd;
using mr_dbbox::dmul;
using mr_dbbox::dsub;
using mr_dbbox::fadd;
using mr_dbbox::fmul;
using mr_dbbox::fsub;

#ifdef __CUDA_ARCH__
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double dsqrt(double a) { return __dsqrt_rn(a); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float fsqrt(float a) { return __fsqrt_rn(a); }
#else
inline double ddiv(double a, double b) { return a / b; }
inline double dsqrt(double a) { return sqrt(a); }
inline float fdiv(float a, float b) { return a / b; }
inline float fsqrt(float a) { return sqrtf(a); }
#endif

// arithmetic in the polygon's dtype, rounded once per operation
__host__ __device__ inline float tmul(float a, float b) { return fmul(a, b); }
__host__ __device__ inline float tadd(float a, float b) { return fadd(a, b); }
__host__ __device__ inline float tsub(float a, float b) { return fsub(a, b); }
__host__ __device__ inline float tsqrt(float a) { return fsqrt(a); }
__host__ __device__ inline double tmul(double a, double b) { return dmul(a, b); }
__host__ __device__ inline double tadd(double a, double b) { return dadd(a, b); }
__host__ __device__ inline double tsub(double a, double b) { return dsub(a, b); }
__host__ __device__ inline double tsqrt(double a) { return dsqrt(a); }

// per-polygon status bits (also the public ones, include/megreader_b200.h)
enum : int {
    kIgnoredIn = 1,        // ignore tag set on input
    kTinyArea = 2,         // |polygon_area| < 1 after clipping
    kSmallText = 4,        // min side < min_text_size
    kShrinkEmpty = 8,      // the shrink has no polygon: mask filled with 0, ignored
    kShrinkPieces = 16,    // the shrink has more than one polygon: the largest is used
    kPadEmpty = 32,        // the pad has no polygon: no border map (the reference raises IndexError)
    kPadPieces = 64,       // the pad has more than one polygon: the largest is used
    kOverflow = 128,       // the clean-up's scratch was too small: treated as an empty result
};

// validate_polygons (make_seg_detection_data.py:79-91) for one [4, 2] polygon q, in place: returns true when |area| < 1
template <class T>
__host__ __device__ inline bool validate_quad(T *q, int H, int W) {
    const T hx = (T)(W - 1), hy = (T)(H - 1);
    for (int i = 0; i < 4; ++i) {           // np.clip(v, 0, w - 1): min(max(v, 0), w - 1)
        T x = q[2 * i], y = q[2 * i + 1];
        x = x < (T)0 ? (T)0 : x;
        x = x > hx ? hx : x;
        y = y < (T)0 ? (T)0 : y;
        y = y > hy ? hy : y;
        q[2 * i] = x;
        q[2 * i + 1] = y;
    }
    T area = (T)0;                          // np.sum of the four edge terms: ((e0 + e1) + e2) + e3, then / 2
    for (int i = 0; i < 4; ++i) {
        const int j = (i + 1) & 3;
        const T e = tmul(tsub(q[2 * j], q[2 * i]), tadd(q[2 * j + 1], q[2 * i + 1]));
        area = i == 0 ? e : tadd(area, e);
    }
    area = tmul(area, (T)0.5);
    if (area > (T)0) {                      // polygons[i][(0, 3, 2, 1), :]
        T t0 = q[2], t1 = q[3];
        q[2] = q[6]; q[3] = q[7];
        q[6] = t0; q[7] = t1;
    }
    const T aa = area < (T)0 ? -area : area;
    return aa < (T)1;
}

// min(height, width) of make_seg_detection_data.py:41-44: the smallest np.linalg.norm of the four sides
template <class T>
__host__ __device__ inline T min_side(const T *q) {
    T m = (T)0;
    for (int i = 0; i < 4; ++i) {
        const int j = (i + 1) & 3;
        const T dx = tsub(q[2 * i], q[2 * j]), dy = tsub(q[2 * i + 1], q[2 * j + 1]);
        const T s = tsqrt(tadd(tmul(dx, dx), tmul(dy, dy)));
        m = i == 0 || s < m ? s : m;
    }
    return m;
}

// ---- the clean-up of one raw offset path (see the top of the file) ----

// Clipper's edge: Bot is the end with the larger Y, Dx = dX / dY (HORIZONTAL for dY = 0)
struct CEdge { int64_t bx, by, tx, ty; double dx; };
constexpr double kHorizontal = -1.0E+40;

__host__ __device__ inline CEdge make_cedge(int64_t x0, int64_t y0, int64_t x1, int64_t y1) {
    CEdge e;
    if (y0 >= y1) { e.bx = x0; e.by = y0; e.tx = x1; e.ty = y1; }
    else { e.bx = x1; e.by = y1; e.tx = x0; e.ty = y0; }
    e.dx = e.by == e.ty ? kHorizontal : ddiv((double)(e.tx - e.bx), (double)(e.ty - e.by));
    return e;
}

__host__ __device__ inline int64_t top_x(const CEdge &e, int64_t y) {
    return y == e.ty ? e.tx : e.bx + clipper_round(dmul(e.dx, (double)(y - e.by)));
}

// IntersectPoint (clipper.cpp) of two crossing edges, e1 the one of lower index on the raw path.  A horizontal edge meets the
// other at (TopX(other, y), y) as ProcessHorizontal does.  The clamp to the bottom of the scan beam uses the higher of the two
// Bot.Y (the scan beam's bottom is not tracked here).
__host__ __device__ inline void clipper_intersect(const CEdge &e1, const CEdge &e2, int64_t &X, int64_t &Y) {
    const bool h1 = e1.dx == kHorizontal, h2 = e2.dx == kHorizontal;
    if (h1 || h2) {
        Y = h1 ? e1.by : e2.by;
        X = top_x(h1 ? e2 : e1, Y);
        return;
    }
    if (e1.dx == 0.) {
        X = e1.bx;
        const double b2 = dsub((double)e2.by, ddiv((double)e2.bx, e2.dx));
        Y = clipper_round(dadd(ddiv((double)X, e2.dx), b2));
    } else if (e2.dx == 0.) {
        X = e2.bx;
        const double b1 = dsub((double)e1.by, ddiv((double)e1.bx, e1.dx));
        Y = clipper_round(dadd(ddiv((double)X, e1.dx), b1));
    } else {
        const double b1 = dsub((double)e1.bx, dmul((double)e1.by, e1.dx));
        const double b2 = dsub((double)e2.bx, dmul((double)e2.by, e2.dx));
        const double q = ddiv(dsub(b2, b1), dsub(e1.dx, e2.dx));
        Y = clipper_round(q);
        X = fabs(e1.dx) < fabs(e2.dx) ? clipper_round(dadd(dmul(e1.dx, q), b1)) : clipper_round(dadd(dmul(e2.dx, q), b2));
    }
    if (Y < e1.ty || Y < e2.ty) {
        Y = e1.ty > e2.ty ? e1.ty : e2.ty;
        X = fabs(e1.dx) < fabs(e2.dx) ? top_x(e1, Y) : top_x(e2, Y);
    }
    const int64_t bot = e1.by < e2.by ? e1.by : e2.by;
    if (Y > bot) {
        Y = bot;
        X = fabs(e1.dx) > fabs(e2.dx) ? top_x(e2, Y) : top_x(e1, Y);
    }
}

__host__ __device__ inline int64_t cross3(int64_t ax, int64_t ay, int64_t bx, int64_t by, int64_t cx, int64_t cy) {
    return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax);
}

__host__ __device__ inline int sgn64(int64_t v) { return (v > 0) - (v < 0); }

// Scratch of clean_offset for a raw path of at most n_cap points, c_cap crossings (2 c_cap split points) and s_cap kept pieces
struct CleanScratch {
    int *cr_e;         // [2 c_cap] edge of each crossing end (two per crossing, one per vertex inside an edge)
    double *cr_t;      // [2 c_cap] parameter along that edge
    int *cr_x, *cr_y;  // [2 c_cap] the rounded crossing point
    int *sx0, *sy0, *sx1, *sy1;  // [s_cap] kept pieces
    unsigned char *used;         // [s_cap]
    int *lx, *ly;                // [s_cap] the loop being traced
    int n_cap, c_cap, s_cap;
};

// class of the turn from u to v with cr = u x v, dt = u . v: 0 right, 1 straight on, 2 left, 3 half turn
__host__ __device__ inline int turn_class(int64_t cr, int64_t dt) { return cr < 0 ? 0 : cr > 0 ? 2 : dt > 0 ? 1 : 3; }

// true when the turn (cr, dt) is strictly sharper to the left (a larger angle in (-pi, pi]) than (cr2, dt2)
__host__ __device__ inline bool turns_left_of(int64_t cr, int64_t dt, int64_t cr2, int64_t dt2) {
    const int a = turn_class(cr, dt), b = turn_class(cr2, dt2);
    if (a != b) return a > b;
    if (a == 2) return dt * cr2 < dt2 * cr;           // angle atan2(cr, dt), cr > 0: larger as dt / cr falls
    if (a == 0) return dt * -cr2 > dt2 * -cr;         // cr < 0: larger as dt / |cr| rises
    return false;
}

// Drops duplicate and collinear points (and spikes) from the loop (lx, ly)[0..m) until none is left; returns the remaining
// count (0 when fewer than three remain) and twice the loop's |area| in *area2.
__host__ __device__ inline int clean_loop(int *lx, int *ly, int m, int64_t *area2) {
    bool changed = true;
    while (changed && m >= 3) {
        changed = false;
        for (int i = 0; i < m && m >= 3; ++i) {
            const int p = i ? i - 1 : m - 1, n = i + 1 < m ? i + 1 : 0;
            if (cross3(lx[p], ly[p], lx[i], ly[i], lx[n], ly[n]) == 0) {
                for (int k = i; k + 1 < m; ++k) { lx[k] = lx[k + 1]; ly[k] = ly[k + 1]; }
                --m;
                --i;
                changed = true;
            }
        }
    }
    if (m < 3) return 0;
    int64_t a = 0;
    for (int i = 0, j = m - 1; i < m; j = i++) a += (int64_t)lx[j] * ly[i] - (int64_t)lx[i] * ly[j];
    *area2 = a < 0 ? -a : a;
    return m;
}

// The clean-up of the raw path (px, py)[0..n): writes the chosen loop to (ox, oy) (at most out_cap points) and returns its
// point count, 0 when there is none; *pieces is the number of loops found; -1 when the scratch is too small.
__host__ __device__ inline int clean_offset(const int *px, const int *py, int n, const CleanScratch &s, int *ox, int *oy,
                                            int out_cap, int *pieces) {
    *pieces = 0;
    if (n < 3) return 0;
    if (n > s.n_cap) return -1;
    // crossings of every pair of non-adjacent raw edges that properly cross (an end on each edge), then every raw vertex that
    // lies inside another edge (one end, on that edge)
    int nc = 0;
    for (int i = 0; i < n; ++i) {
        const int i1 = i + 1 < n ? i + 1 : 0;
        for (int j = i + 2; j < n; ++j) {
            const int j1 = j + 1 < n ? j + 1 : 0;
            if (j1 == i) continue;
            const int64_t d1 = cross3(px[i], py[i], px[i1], py[i1], px[j], py[j]);
            const int64_t d2 = cross3(px[i], py[i], px[i1], py[i1], px[j1], py[j1]);
            const int64_t d3 = cross3(px[j], py[j], px[j1], py[j1], px[i], py[i]);
            const int64_t d4 = cross3(px[j], py[j], px[j1], py[j1], px[i1], py[i1]);
            if (sgn64(d1) * sgn64(d2) >= 0 || sgn64(d3) * sgn64(d4) >= 0) continue;
            if (nc + 2 > 2 * s.c_cap) return -1;
            int64_t X, Y;
            clipper_intersect(make_cedge(px[i], py[i], px[i1], py[i1]), make_cedge(px[j], py[j], px[j1], py[j1]), X, Y);
            // parameters of the exact crossing along both edges: d3 / (d3 - d4) along i, d1 / (d1 - d2) along j
            s.cr_e[nc] = i;
            s.cr_t[nc] = ddiv((double)d3, (double)(d3 - d4));
            s.cr_e[nc + 1] = j;
            s.cr_t[nc + 1] = ddiv((double)d1, (double)(d1 - d2));
            s.cr_x[nc] = s.cr_x[nc + 1] = (int)X;
            s.cr_y[nc] = s.cr_y[nc + 1] = (int)Y;
            nc += 2;
        }
    }
    for (int i = 0; i < n; ++i) {
        const int i1 = i + 1 < n ? i + 1 : 0;
        const int64_t ex = px[i1] - px[i], ey = py[i1] - py[i], len2 = ex * ex + ey * ey;
        for (int v = 0; v < n; ++v) {
            if (cross3(px[i], py[i], px[i1], py[i1], px[v], py[v]) != 0) continue;
            const int64_t dot = (px[v] - px[i]) * ex + (py[v] - py[i]) * ey;
            if (dot <= 0 || dot >= len2) continue;
            if (nc + 1 > 2 * s.c_cap) return -1;
            s.cr_e[nc] = i;
            s.cr_t[nc] = ddiv((double)dot, (double)len2);
            s.cr_x[nc] = px[v];
            s.cr_y[nc] = py[v];
            nc += 1;
        }
    }
    // the pieces of every edge, in order along it; a piece is kept when the winding just left of it is 1
    const double PI = 3.141592653589793238, TWO_PI = PI * 2;
    int ns = 0;
    for (int i = 0; i < n; ++i) {
        const int i1 = i + 1 < n ? i + 1 : 0;
        int ax = px[i], ay = py[i];
        double ta = 0.;
        int last = -1;                      // crossing end taken last: the next is the least (t, index) after it
        for (;;) {
            int best = -1;
            for (int k = 0; k < nc; ++k) {
                if (s.cr_e[k] != i) continue;
                const bool after = last < 0 || s.cr_t[k] > s.cr_t[last] || (s.cr_t[k] == s.cr_t[last] && k > last);
                if (after && (best < 0 || s.cr_t[k] < s.cr_t[best] || (s.cr_t[k] == s.cr_t[best] && k < best))) best = k;
            }
            const int bx = best < 0 ? px[i1] : s.cr_x[best], by = best < 0 ? py[i1] : s.cr_y[best];
            const double tb = best < 0 ? 1. : s.cr_t[best];
            if (ax != bx || ay != by) {
                // winding at the middle of the exact piece: the angle the rest of the path sweeps around it, plus pi
                const double tm = dmul(dadd(ta, tb), 0.5);
                const double mx = dadd((double)px[i], dmul(tm, (double)(px[i1] - px[i])));
                const double my = dadd((double)py[i], dmul(tm, (double)(py[i1] - py[i])));
                double th = 0.;
                for (int j = 0; j < n; ++j) {
                    if (j == i) continue;
                    const int j1 = j + 1 < n ? j + 1 : 0;
                    const double ux = dsub((double)px[j], mx), uy = dsub((double)py[j], my);
                    const double vx = dsub((double)px[j1], mx), vy = dsub((double)py[j1], my);
                    th = dadd(th, atan2(dsub(dmul(ux, vy), dmul(uy, vx)), dadd(dmul(ux, vx), dmul(uy, vy))));
                }
                const double w = floor(dadd(ddiv(dadd(th, PI), TWO_PI), 0.5));
                if (w == 1.) {
                    if (ns >= s.s_cap) return -1;
                    s.sx0[ns] = ax; s.sy0[ns] = ay; s.sx1[ns] = bx; s.sy1[ns] = by;
                    s.used[ns] = 0;
                    ++ns;
                }
            }
            if (best < 0) break;
            ax = bx; ay = by; ta = tb; last = best;
        }
    }
    // chain the kept pieces into loops; keep the one of largest |area|
    int64_t best_area = -1;
    int out_n = 0;
    for (int st = 0; st < ns; ++st) {
        if (s.used[st]) continue;
        int m = 0, cur = st;
        while (cur >= 0) {
            s.used[cur] = 1;
            if (m >= s.s_cap) return -1;
            s.lx[m] = s.sx0[cur]; s.ly[m] = s.sy0[cur]; ++m;
            const int64_t ux = s.sx1[cur] - s.sx0[cur], uy = s.sy1[cur] - s.sy0[cur];
            int nxt = -1;
            int64_t ncr = 0, ndt = 0;
            for (int k = 0; k < ns; ++k) {
                if (s.used[k] || s.sx0[k] != s.sx1[cur] || s.sy0[k] != s.sy1[cur]) continue;
                const int64_t vx = s.sx1[k] - s.sx0[k], vy = s.sy1[k] - s.sy0[k];
                const int64_t cr = ux * vy - uy * vx, dt = ux * vx + uy * vy;
                if (nxt < 0 || turns_left_of(cr, dt, ncr, ndt)) { nxt = k; ncr = cr; ndt = dt; }
            }
            cur = nxt;
        }
        int64_t area2 = 0;
        m = clean_loop(s.lx, s.ly, m, &area2);
        if (m == 0) continue;
        ++*pieces;
        if (area2 > best_area) {
            best_area = area2;
            out_n = m;
            if (out_n > out_cap) return -1;
            for (int k = 0; k < out_n; ++k) { ox[k] = s.lx[k]; oy[k] = s.ly[k]; }
        }
    }
    return out_n;
}

// ---- cv2.fillPoly of one polygon, pixel by pixel ----
// FillEdgeCollection walks the rows keeping the active edges (y0 <= y < y1) sorted by x and advancing each by dx per row,
// and fills between the 1st and 2nd, 3rd and 4th, ... of them.  So at row y edge e sits at x + (y - y0) dx, and pixel X is
// set iff an odd number of those positions are < X << 16, or one is == X << 16.  Pixels are therefore independent.
using mr_dbbox::PolyEdge;

// the bounds FillEdgeCollection tests before filling anything (false when the edges lie wholly off the image, or there are
// fewer than two), and the rows [y_lo, y_hi) and columns [x_lo, x_hi] the fill can touch.  e[0..n) holds one entry per
// polygon edge; horizontal ones have y0 >= y1.
__host__ __device__ inline bool fill_bounds(const PolyEdge *e, int n, int width, int height, int &y_lo, int &y_hi, int &x_lo,
                                            int &x_hi) {
    int ne = 0;
    for (int i = 0; i < n; ++i) ne += e[i].y0 < e[i].y1;
    if (ne < 2) return false;
    int y_max = INT32_MIN, y_min = INT32_MAX;
    int64_t x_max = -1, x_min = INT64_MAX;
    for (int i = 0; i < n; ++i) {
        if (e[i].y0 >= e[i].y1) continue;   // horizontal: no PolyEdge
        const int64_t x1 = e[i].x + (int64_t)(e[i].y1 - e[i].y0) * e[i].dx;
        y_min = e[i].y0 < y_min ? e[i].y0 : y_min;
        y_max = e[i].y1 > y_max ? e[i].y1 : y_max;
        x_min = e[i].x < x_min ? e[i].x : x_min;
        x_max = e[i].x > x_max ? e[i].x : x_max;
        x_min = x1 < x_min ? x1 : x_min;
        x_max = x1 > x_max ? x1 : x_max;
    }
    if (y_max < 0 || y_min >= height || x_max < 0 || x_min >= ((int64_t)width << 16)) return false;
    y_lo = y_min > 0 ? y_min : 0;                       // the rows and columns the fill can touch
    y_hi = y_max < height ? y_max : height;
    x_lo = (int)(x_min > 0 ? x_min >> 16 : 0);
    x_hi = (int)((x_max >> 16) < width - 1 ? (x_max >> 16) : width - 1);
    return true;
}

__host__ __device__ inline bool pixel_filled(const PolyEdge *e, int n, int X, int y) {
    const int64_t v = (int64_t)X << 16;
    int lt = 0;
    bool eq = false;
    for (int i = 0; i < n; ++i) {
        if (y < e[i].y0 || y >= e[i].y1) continue;
        const int64_t x = e[i].x + (int64_t)(y - e[i].y0) * e[i].dx;
        lt += x < v;
        eq |= x == v;
    }
    return (lt & 1) || eq;
}

// ---- MakeBorderMap.distance (make_border_map.py:97-121) at one pixel for one edge, float64 without FMA ----
// (xs, ys) the pixel and (ax, ay), (bx, by) the edge ends in the shifted frame; sd is np.square(dx) + np.square(dy) of the
// edge, computed in the polygon's dtype.  NaN where the reference's is.
__host__ __device__ inline double edge_distance(double xs, double ys, double ax, double ay, double bx, double by, double sd) {
    const double u = dsub(xs, ax), v = dsub(ys, ay), p = dsub(xs, bx), q = dsub(ys, by);
    const double sd1 = dadd(dmul(u, u), dmul(v, v)), sd2 = dadd(dmul(p, p), dmul(q, q));
    const double cosin = ddiv(dsub(dsub(sd, sd1), sd2), dmul(2., dsqrt(dmul(sd1, sd2))));
    double ss = dsub(1., dmul(cosin, cosin));
    if (ss != ss) ss = 0.;                  // np.nan_to_num
    else if (ss == INFINITY) ss = 1.7976931348623157e308;
    else if (ss == -INFINITY) ss = -1.7976931348623157e308;
    double r = dsqrt(ddiv(dmul(dmul(sd1, sd2), ss), sd));
    if (cosin < 0.) r = dsqrt(sd1 < sd2 ? sd1 : sd2);
    return r;
}

// 1 - min_i clip(distance_i / distance, 0, 1) of one pixel over the quad's four edges, each rounded to float32; NaN when
// any edge's is (np.min propagates it)
template <class T>
__host__ __device__ inline float border_value(const T *q, double xmin, double ymin, double xs, double ys, double distance) {
    float m = 0.f;
    for (int i = 0; i < 4; ++i) {
        const int j = (i + 1) & 3;
        // polygon[:, 0] - xmin, stored back into the polygon's dtype
        const T ax = (T)dsub((double)q[2 * i], xmin), ay = (T)dsub((double)q[2 * i + 1], ymin);
        const T bx = (T)dsub((double)q[2 * j], xmin), by = (T)dsub((double)q[2 * j + 1], ymin);
        const T dx = tsub(ax, bx), dy = tsub(ay, by);
        const double sd = (double)tadd(tmul(dx, dx), tmul(dy, dy));
        double d = ddiv(edge_distance(xs, ys, (double)ax, (double)ay, (double)bx, (double)by, sd), distance);
        if (d == d) d = d < 0. ? 0. : d > 1. ? 1. : d;
        const float f = (float)d;
        if (f != f) return f;
        m = i == 0 || f < m ? f : m;
    }
    return fsub(1.f, m);
}

// cv2.fillPoly(img, [poly], value) of the n-point integer polygon (xs, ys): edge i joins point i - 1 to point i.  The
// PolyEdge of edge i, with y0 = y1 = 0 for a horizontal one; visits the pixels of its line.
template <class Visit>
__host__ __device__ inline PolyEdge fill_edge(const int *xs, const int *ys, int n, int i, int width, int height, Visit visit) {
    const int k = i ? i - 1 : n - 1;
    mr_dbbox::L2 a, b;
    bool draw;
    PolyEdge e;
    if (!mr_dbbox::poly_edge(xs[k], ys[k], xs[i], ys[i], width, height, a, b, draw, e)) { e.y0 = e.y1 = 0; e.x = e.dx = 0; }
    if (draw) mr_dbbox::draw_line(a, b, visit);
    return e;
}

// ---- one polygon of MakeSegDetectionData.process and MakeBorderMap.draw_border_map ----

// Scratch sizes for images of at most `dim` pixels a side: the raw path (Clipper's arc steps for a distance up to `dim`,
// plus three points per corner), crossings and kept pieces.  The shrunk and padded polygons have at most `pieces` points.
struct Caps { int raw, cross, pieces; };
__host__ __device__ inline Caps caps_for(int dim) {
    Caps c;
    c.raw = mr_dbbox::unclip_max_points((double)dim);
    c.cross = 2 * c.raw + 64;
    c.pieces = c.raw + 2 * c.cross;
    return c;
}

// Validates the quad q in place and computes its shrunk polygon (sx, sy)[0..*n_shrink) and padded polygon
// (px, py)[0..*n_pad), both with at most caps.pieces points.  Returns the status bits; the polygon is ignored afterwards
// when any of kIgnoredIn, kTinyArea, kSmallText, kShrinkEmpty or kOverflow (before the pad) is set.
template <class T>
__host__ __device__ inline int polygon_targets(T *q, bool ignore_in, int H, int W, double shrink_k, double min_text, const Caps &c,
                                               int *rx, int *ry, const CleanScratch &s, int *sx, int *sy, int *n_shrink, int *px,
                                               int *py, int *n_pad, double *distance) {
    int status = ignore_in ? kIgnoredIn : 0;
    *n_shrink = *n_pad = 0;
    *distance = 0.;
    if (validate_quad(q, H, W)) status |= kTinyArea;
    if (status) return status;
    if ((double)min_side(q) < min_text) return status | kSmallText;
    double area, length;
    mr_dbbox::ring_area_length(q, area, length);
    const double d = ddiv(dmul(area, shrink_k), length);
    *distance = d;
    int pieces = 0;
    int n = mr_dbbox::unclip_offset(q, -d, rx, ry, c.raw);
    n = n < 0 ? -1 : clean_offset(rx, ry, n, s, sx, sy, c.pieces, &pieces);
    if (n < 0) return status | kOverflow;
    if (n == 0) return status | kShrinkEmpty;
    if (pieces > 1) status |= kShrinkPieces;
    *n_shrink = n;
    n = mr_dbbox::unclip_offset(q, d, rx, ry, c.raw);
    n = n < 0 ? -1 : clean_offset(rx, ry, n, s, px, py, c.pieces, &pieces);
    if (n < 0) return status | kOverflow | kPadEmpty;
    if (n == 0) return status | kPadEmpty;
    if (pieces > 1) status |= kPadPieces;
    *n_pad = n;
    return status;
}

__host__ __device__ inline bool status_ignored(int status) {
    return (status & (kIgnoredIn | kTinyArea | kSmallText | kShrinkEmpty)) || ((status & kOverflow) && !(status & kPadEmpty));
}

}  // namespace mr_dbtgt
