// Host-side harness: runs the PRODUCT's per-contour routines (megreader_b200/csrc/db_boxes_core.cuh, the code the CUDA kernels in
// db_boxes.cu execute) on the CPU, so that tests can compare them with cv2 without a GPU.  Built on demand by
// tests/test_db_boxes_cpu.py with g++ (no CUDA involved).
#include <vector>

#include "db_boxes_core.cuh"

extern "C" {

// Traces the contours whose start pixels are given (starts[2i] = raster index, starts[2i + 1] = 1 for a hole border) into
// points (x, y pairs, at most `capacity` points); offsets[i] .. offsets[i + 1] are the points of contour i.  Returns the total
// number of points (which may exceed `capacity`: points past it are not written).
long long host_trace_contours(const unsigned char *bm, int H, int W, const long long *starts, int n, int *points, long long capacity,
                              long long *offsets) {
    long long total = 0;
    for (int i = 0; i < n; ++i) {
        offsets[i] = total;
        const int x0 = (int)(starts[2 * i] % W), y0 = (int)(starts[2 * i] / W);
        mr_dbbox::trace_border(bm, H, W, x0, y0, starts[2 * i + 1] != 0, [&](int x, int y) {
            if (total < capacity) { points[2 * total] = x; points[2 * total + 1] = y; }
            ++total;
        });
    }
    offsets[n] = total;
    return total;
}

}

extern "C" int host_convex_hull(const int *xy, int n, int *hull) {
    std::vector<int> o(n), st(n + 2);
    return mr_dbbox::convex_hull((const mr_dbbox::Pt *)xy, n, o.data(), st.data(), hull);
}

// cv2.minAreaRect(points) for int32 points: out = (cx, cy, w, h, angle)
extern "C" void host_min_area_rect(const int *xy, int n, float *out) {
    std::vector<int> o(n), st(n + 2), hull(n);
    const int k = mr_dbbox::convex_hull((const mr_dbbox::Pt *)xy, n, o.data(), st.data(), hull.data());
    std::vector<float> qx(k), qy(k), vx(k), vy(k), inv(k);
    for (int i = 0; i < k; ++i) { qx[i] = (float)xy[2 * hull[i]]; qy[i] = (float)xy[2 * hull[i] + 1]; }
    const mr_dbbox::Rect r = mr_dbbox::min_area_rect_hull(qx.data(), qy.data(), k, vx.data(), vy.data(), inv.data());
    out[0] = r.cx; out[1] = r.cy; out[2] = r.w; out[3] = r.h; out[4] = r.angle;
}

// get_mini_boxes(contour) for int32 points: box[8] and the return value sside
extern "C" float host_mini_box(const int *xy, int n, float *box) {
    float r[5];
    host_min_area_rect(xy, n, r);
    return mr_dbbox::mini_box(mr_dbbox::Rect{r[0], r[1], r[2], r[3], r[4]}, box);
}

// cv2.fillPoly(mask, [quad], 1) on a zero width x height uint8 mask
extern "C" void host_fill_quad(const int *quad, int width, int height, unsigned char *mask) {
    mr_dbbox::fill_quad(quad, width, height, height, [&](int x, int y) { mask[(int64_t)y * width + x] = 1; });
}

// box_score_fast(pred, box) for an H x W fp32 map and a [4, 2] fp32 box
extern "C" double host_box_score(const float *pred, int H, int W, const float *box) { return mr_dbbox::box_score(pred, H, W, box); }

// the unclip of a [4, 2] fp32 box: distance (out) and the offset path into xy (at most cap points); returns the point count
extern "C" int host_unclip(const float *box, double *distance, int *xy, int cap) {
    *distance = mr_dbbox::unclip_distance(box);
    std::vector<int> x(cap), y(cap);
    const int n = mr_dbbox::unclip_offset(box, *distance, x.data(), y.data(), cap);
    for (int i = 0; i < n; ++i) { xy[2 * i] = x[i]; xy[2 * i + 1] = y[i]; }
    return n;
}

// rescale of one coordinate
extern "C" int host_rescale(float v, int size, int dest) { return mr_dbbox::rescale(v, size, dest); }
