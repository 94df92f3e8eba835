// Host-side harness: runs the PRODUCT's per-polygon and per-pixel routines of the DB targets
// (megreader_b200/csrc/db_targets_core.cuh, the code the CUDA kernels in db_targets.cu execute) on the CPU, so that tests can
// compare them with cv2, numpy and the oracle without a GPU.  Built on demand by tests/test_db_targets_cpu.py with g++.
#include <vector>

#include "db_targets_core.cuh"

using namespace mr_dbtgt;

extern "C" {

// cv2.fillPoly(mask, [poly], 1) of the n-point int32 polygon xy on a zero width x height uint8 mask, pixel by pixel
void host_fill_poly(const int *xy, int n, int width, int height, unsigned char *mask) {
    std::vector<int> xs(n), ys(n);
    for (int i = 0; i < n; ++i) { xs[i] = xy[2 * i]; ys[i] = xy[2 * i + 1]; }
    std::vector<PolyEdge> e(n);
    for (int i = 0; i < n; ++i)
        e[i] = fill_edge(xs.data(), ys.data(), n, i, width, height, [&](int x, int y) { mask[(int64_t)y * width + x] = 1; });
    int y_lo, y_hi, x_lo, x_hi;
    if (!fill_bounds(e.data(), n, width, height, y_lo, y_hi, x_lo, x_hi)) return;
    for (int y = y_lo; y < y_hi; ++y)
        for (int x = x_lo; x <= x_hi; ++x)
            if (pixel_filled(e.data(), n, x, y)) mask[(int64_t)y * width + x] = 1;
}

// MakeBorderMap.distance for the count pixels (xs, ys) and one edge
void host_edge_distance(const double *xs, const double *ys, int64_t count, double ax, double ay, double bx, double by, double sd,
                        double *out) {
    for (int64_t i = 0; i < count; ++i) out[i] = edge_distance(xs[i], ys[i], ax, ay, bx, by, sd);
}

// The clean-up of a raw path xy[0..n): the chosen loop into out (at most cap points); returns its count, *pieces the loops
int host_clean_offset(const int *xy, int n, int *out, int cap, int *pieces) {
    const int c_cap = 2 * n + 64, s_cap = n + 2 * c_cap;
    std::vector<int> px(n), py(n), cre(2 * c_cap), crx(2 * c_cap), cry(2 * c_cap), s4(4 * s_cap), l(2 * s_cap), o(2 * cap);
    std::vector<double> crt(2 * c_cap);
    std::vector<unsigned char> used(s_cap);
    for (int i = 0; i < n; ++i) { px[i] = xy[2 * i]; py[i] = xy[2 * i + 1]; }
    CleanScratch s{cre.data(), crt.data(), crx.data(), cry.data(), s4.data(), s4.data() + s_cap, s4.data() + 2 * s_cap,
                   s4.data() + 3 * s_cap, used.data(), l.data(), l.data() + s_cap, n, c_cap, s_cap};
    const int m = clean_offset(px.data(), py.data(), n, s, o.data(), o.data() + cap, cap, pieces);
    for (int i = 0; i < m; ++i) { out[2 * i] = o[i]; out[2 * i + 1] = o[cap + i]; }
    return m;
}

// The raw offset path of a [4, 2] quad (float64 corners) for delta into xy (at most cap points); returns the count
int host_raw_offset(const double *quad, double delta, int *xy, int cap) {
    std::vector<int> x(cap), y(cap);
    const int n = mr_dbbox::unclip_offset(quad, delta, x.data(), y.data(), cap);
    for (int i = 0; i < n; ++i) { xy[2 * i] = x[i]; xy[2 * i + 1] = y[i]; }
    return n;
}

}  // extern "C"

// Both processes for one H x W image, sequentially, with the kernels' routines: polygons [n, 4, 2] (float32 when f32, else
// float64) are validated in place; ignore [n] is updated; status [n]; maps as the device call writes them.
template <class T>
static void make_targets(T *polys, int n, unsigned char *ignore, int H, int W, double shrink_k, double min_text, float scale,
                         float lo, float *gt, float *mask, float *thresh_map, float *thresh_mask, int *status) {
    const Caps c = caps_for(H > W ? H : W);
    std::vector<int> rx(c.raw), ry(c.raw), cre(2 * c.cross), crx(2 * c.cross), cry(2 * c.cross), s4(4 * c.pieces),
        l(2 * c.pieces), sh(2 * c.pieces), pad(2 * c.pieces);
    std::vector<double> crt(2 * c.cross);
    std::vector<unsigned char> used(c.pieces);
    const int S = c.pieces;
    CleanScratch s{cre.data(), crt.data(), crx.data(), cry.data(), s4.data(), s4.data() + S, s4.data() + 2 * S, s4.data() + 3 * S,
                   used.data(), l.data(), l.data() + S, c.raw, c.cross, S};
    for (int64_t i = 0; i < (int64_t)H * W; ++i) { gt[i] = 0.f; mask[i] = 1.f; thresh_map[i] = 0.f; thresh_mask[i] = 0.f; }
    auto fill = [&](const int *xs, const int *ys, int m, float *img, float value) {
        std::vector<PolyEdge> e(m);
        auto set = [&](int x, int y) { img[(int64_t)y * W + x] = value; };
        for (int i = 0; i < m; ++i) e[i] = fill_edge(xs, ys, m, i, W, H, set);
        int y_lo, y_hi, x_lo, x_hi;
        if (!fill_bounds(e.data(), m, W, H, y_lo, y_hi, x_lo, x_hi)) return;
        for (int y = y_lo; y < y_hi; ++y)
            for (int x = x_lo; x <= x_hi; ++x)
                if (pixel_filled(e.data(), m, x, y)) set(x, y);
    };
    for (int p = 0; p < n; ++p) {
        T *q = polys + 8 * p;
        int ns, np_;
        double d;
        status[p] = polygon_targets(q, ignore[p] != 0, H, W, shrink_k, min_text, c, rx.data(), ry.data(), s, sh.data(), sh.data() + S,
                                    &ns, pad.data(), pad.data() + S, &np_, &d);
        const bool ign = status_ignored(status[p]);
        ignore[p] = ign;
        if (ign) {
            int qx[4], qy[4];
            for (int k = 0; k < 4; ++k) { qx[k] = (int)q[2 * k]; qy[k] = (int)q[2 * k + 1]; }
            fill(qx, qy, 4, mask, 0.f);
            continue;
        }
        if (ns) fill(sh.data(), sh.data() + S, ns, gt, 1.f);
        if (!np_) continue;
        fill(pad.data(), pad.data() + S, np_, thresh_mask, 1.f);
        int xmin = pad[0], xmax = pad[0], ymin = pad[S], ymax = pad[S];
        for (int k = 1; k < np_; ++k) {
            xmin = std::min(xmin, pad[k]); xmax = std::max(xmax, pad[k]);
            ymin = std::min(ymin, pad[S + k]); ymax = std::max(ymax, pad[S + k]);
        }
        const int x0 = std::min(std::max(0, xmin), W - 1), x1 = std::min(std::max(0, xmax), W - 1);
        const int y0 = std::min(std::max(0, ymin), H - 1), y1 = std::min(std::max(0, ymax), H - 1);
        for (int y = y0; y <= y1; ++y)
            for (int x = x0; x <= x1; ++x) {
                const float v = border_value(q, (double)xmin, (double)ymin, (double)(x - xmin), (double)(y - ymin), d);
                float &cv = thresh_map[(int64_t)y * W + x];
                if (v == v && v > cv) cv = v;
            }
    }
    for (int64_t i = 0; i < (int64_t)H * W; ++i) thresh_map[i] = thresh_map[i] * scale + lo;
}

extern "C" void host_make_targets(void *polys, int f32, int n, unsigned char *ignore, int H, int W, double shrink_k, double min_text,
                                  float scale, float lo, float *gt, float *mask, float *thresh_map, float *thresh_mask, int *status) {
    if (f32)
        make_targets((float *)polys, n, ignore, H, W, shrink_k, min_text, scale, lo, gt, mask, thresh_map, thresh_mask, status);
    else
        make_targets((double *)polys, n, ignore, H, W, shrink_k, min_text, scale, lo, gt, mask, thresh_map, thresh_mask, status);
}
