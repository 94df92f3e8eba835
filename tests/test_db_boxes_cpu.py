"""CPU: the PRODUCT's per-candidate routines (megreader_b200/csrc/db_boxes_core.cuh -- the code the CUDA kernels of
csrc/db_boxes.cu run) compiled for the host by tests/host_harness/db_boxes_core_host.cpp and compared with cv2:
  * the border tracer with cv2.findContours(RETR_LIST, CHAIN_APPROX_NONE) (seg_detector_representer.py:73-75) array for array,
    and the start-pixel rule the kernels implement (component roots, enclosed holes, descending raster order);
  * convex hull, rotating calipers, box corners and their order with cv2.convexHull / cv2.minAreaRect / cv2.boxPoints and the
    reference's get_mini_boxes (:125-145) on every one of those contours, with the one counted class of differences;
  * the quad fill with cv2.fillPoly on random int32 quads, and the box score with the reference's box_score_fast (:156-168);
and the C-ABI's argument checks."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.db_boxes_cases import adversarial_bitmaps, box_score_fast, cv2_contours, get_mini_boxes, prob_maps, random_bitmaps

cv2 = pytest.importorskip("cv2")
ndimage = pytest.importorskip("scipy.ndimage")

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("harness") / "libdb_boxes_core_host.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                           "-I", os.path.join(HERE, "..", "megreader_b200", "csrc"),
                           os.path.join(HERE, "host_harness", "db_boxes_core_host.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    lib.host_trace_contours.restype = ctypes.c_longlong
    lib.host_mini_box.restype = ctypes.c_float
    lib.host_box_score.restype = ctypes.c_double
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def start_pixels(bm):
    """(raster index, is hole) of every contour start in descending raster order: the first pixel of each 8-connected
    foreground component, and the pixel left of the first pixel of each 4-connected background component off the frame"""
    out = []
    fg, _ = ndimage.label(bm, np.ones((3, 3), int))
    bg, _ = ndimage.label(bm == 0)
    for lab, hole in ((fg, 0), (bg, 1)):
        flat = lab.ravel()
        nz = np.flatnonzero(flat)
        ids, first = np.unique(flat[nz], return_index=True)
        for i, f in zip(ids, nz[first]):
            if hole:
                m = lab == i
                if m[0].any() or m[-1].any() or m[:, 0].any() or m[:, -1].any():
                    continue
                f -= 1
            out.append((int(f), hole))
    out.sort(key=lambda t: -t[0])
    return np.array(out, np.int64).reshape(-1, 2)


def trace(lib, bm, starts):
    H, W = bm.shape
    bm = np.ascontiguousarray(bm != 0, np.uint8)
    starts = np.ascontiguousarray(starts, np.int64)
    cap = 4 * H * W
    pts = np.zeros((cap, 2), np.int32)
    off = np.zeros(len(starts) + 1, np.int64)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    total = lib.host_trace_contours(p(bm), H, W, p(starts), len(starts), p(pts), ctypes.c_longlong(cap), p(off))
    assert total <= cap, "more than 4 points per pixel"
    return [pts[off[i]:off[i + 1]] for i in range(len(starts))]


def check_against_cv2(lib, bm):
    want = cv2_contours(bm)
    st = start_pixels(bm)
    W = bm.shape[1]
    # the start rule the kernels rely on: cv2's contour i begins at start pixel i
    assert len(want) == len(st)
    assert all(tuple(c[0, 0]) == (s % W, s // W) for c, (s, _) in zip(want, st))
    got = trace(lib, bm, st)
    for i, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w.reshape(-1, 2)), (i, g.tolist(), w.reshape(-1, 2).tolist())


def test_tracer_equals_cv2_on_random_bitmaps(harness):
    bms = random_bitmaps(2024, 3000)
    for bm in bms:
        check_against_cv2(harness, bm)
    assert sum(len(start_pixels(b)) for b in bms) > 30000


@pytest.mark.parametrize("name", sorted(adversarial_bitmaps()))
def test_tracer_equals_cv2_on_adversarial_bitmaps(harness, name):
    bm = adversarial_bitmaps()[name]
    check_against_cv2(harness, bm)
    for k in range(1, 4):                             # every orientation of the same structure
        check_against_cv2(harness, np.ascontiguousarray(np.rot90(bm, k)))


def test_holes_yield_their_own_contours(harness):
    """nested structure: outer ring, its hole, the island inside, the island's hole -- four contours, two of them holes"""
    bm = adversarial_bitmaps()["nested_holes_and_islands"]
    st = start_pixels(bm)
    assert len(cv2_contours(bm)) == 4 and st[:, 1].tolist() == [1, 0, 1, 0]


def all_contours():
    return [np.ascontiguousarray(c.reshape(-1, 2), np.int32)
            for bm in random_bitmaps(5, 3000) + list(adversarial_bitmaps().values()) for c in cv2_contours(bm)]


def test_convex_hull_vs_cv2(harness):
    """The hull's vertices, orientation and cyclic order equal cv2.convexHull(clockwise=False) on every contour.  Where a
    contour passes a hull vertex more than once, which of the equal points cv2 reports (and so where its index-ordered output
    starts) is not reproduced on ~0.5 % of the contours; minAreaRect does not depend on it on any of them."""
    starts_differ = 0
    cs = all_contours()
    for c in cs:
        h = np.zeros(len(c), np.int32)
        k = harness.host_convex_hull(_p(c), len(c), _p(h))
        got, want = c[h[:k]], cv2.convexHull(c, clockwise=False).reshape(-1, 2)
        assert len(got) == len(want)
        shift = [s for s in range(len(got)) if np.array_equal(np.roll(got, -s, axis=0), want)]
        assert shift, (c.tolist(), got.tolist(), want.tolist())
        starts_differ += shift[0] != 0
    assert len(cs) > 50000 and starts_differ <= 0.01 * len(cs)


def test_min_area_rect_and_mini_boxes_vs_cv2(harness):
    """cv2.minAreaRect (centre, size, angle in [-90, 0)) and get_mini_boxes' corners and sside, bit for bit, except one
    counted class: rectangles that several hull edges give (parallel edges, or the sides of a 45-degree rectangle), where the
    calipers' float tie goes to another edge than cv2's -- the same angle, centre and size a few float ulps apart (49 of
    ~54,000 contours)."""
    ties = 0
    cs = all_contours()
    for c in cs:
        r = np.zeros(5, np.float32)
        harness.host_min_area_rect(_p(c), len(c), _p(r))
        box = np.zeros(8, np.float32)
        sside = harness.host_mini_box(_p(c), len(c), _p(box))
        (cx, cy), (w, h), a = cv2.minAreaRect(c)
        want = np.array([cx, cy, w, h, a], np.float32)
        wbox, wside = get_mini_boxes(c)
        exact = np.array_equal(r, want)
        if not exact:
            assert r[4] == want[4], (c.tolist(), r.tolist(), want.tolist())
            assert np.abs(r - want).max() <= 4 * np.spacing(np.abs(want).max()), (r.tolist(), want.tolist())
            assert np.abs(box.reshape(4, 2) - wbox).max() <= 4 * np.spacing(np.abs(wbox).max())
            ties += 1
        else:
            assert np.array_equal(box.reshape(4, 2), wbox) and np.float32(sside) == np.float32(wside), c.tolist()
    assert ties <= 0.002 * len(cs), ties


def random_quads(seed, n):
    """(quad int32 [4, 2], width, height): inside, negative, far outside, degenerate (repeated points, lines), self-intersecting
    and 1-pixel-thin quads"""
    rng = np.random.RandomState(seed)
    for i in range(n):
        W, H = (int(v) for v in rng.randint(1, 30, 2))
        kind = i % 5
        if kind == 0:
            q = rng.randint(-5, max(W, H) + 5, (4, 2))
        elif kind == 1:
            q = rng.randint(0, 6, (4, 2))
        elif kind == 2:
            q = rng.randint(-40, 60, (4, 2))
        elif kind == 3:
            q = np.repeat(rng.randint(-3, 20, (1, 2)), 4, 0) + rng.randint(0, 2, (4, 2))
        else:
            a, b = rng.randint(-3, 25, (2, 2))
            q = np.array([a, b, b + [0, 1], a + [0, 1]]) if rng.rand() < 0.5 else np.array([a, b, b + [1, 0], a + [1, 0]])
        yield np.ascontiguousarray(q, np.int32), W, H


def test_fill_quad_equals_cv2_fillpoly(harness):
    n = 0
    for q, W, H in random_quads(11, 12000):
        want = np.zeros((H, W), np.uint8)
        cv2.fillPoly(want, q.reshape(1, 4, 2), 1)
        got = np.zeros((H, W), np.uint8)
        harness.host_fill_quad(_p(q), W, H, _p(got))
        assert np.array_equal(got, want), (q.tolist(), W, H)
        n += 1
    assert n >= 10000


def test_box_score_equals_box_score_fast(harness):
    """the mini boxes of DB-like maps (boxes at the borders included) and random boxes partly or wholly outside the map, on
    small maps and on one wider than a mask band (8192 columns: a band is then one row in pieces)"""
    rng = np.random.RandomState(3)
    wide = np.ascontiguousarray(rng.uniform(0, 1, (1, 1, 6, 9000)).astype(np.float32))
    m = wide[0, 0]
    for b in list(rng.uniform(-50, 9050, (20, 4, 2)) * [1, 0.001]) + [np.array([[-5, 1], [8800, 0.5], [8990, 4.2], [10, 5]])]:
        b = np.ascontiguousarray(b, np.float32)
        assert harness.host_box_score(_p(m), 6, 9000, _p(b)) == box_score_fast(m, b), b.tolist()
    for m in list(prob_maps(13, 3, 97, 131)) + list(prob_maps(14, 1, 40, 700)):
        m = np.ascontiguousarray(m[0])
        H, W = m.shape
        boxes = [get_mini_boxes(c)[0] for c in cv2_contours(m > 0.3)]
        boxes += list(rng.uniform(-20, 150, (1000, 4, 2)))
        boxes += list(rng.uniform(0, 120, (1000, 1, 2)) + rng.uniform(-2, 2, (1000, 4, 2)))
        for b in boxes:
            b = np.ascontiguousarray(b, np.float32)
            assert harness.host_box_score(_p(m), H, W, _p(b)) == box_score_fast(m, b), b.tolist()


def test_capi_argument_checks_without_gpu():
    from megreader_b200 import _lib
    from megreader_b200 import build
    build.build()
    L = _lib.lib()
    r = lambda n: -(-n // 256) * 256  # noqa: E731
    for N, H, W, maxc in ((1, 1, 1, 0), (4, 576, 1024, 1000), (3, 33, 47, 100), (16, 640, 640, 1)):
        HW = H * W
        want = 2 * r(N * HW) + r(4 * N * HW) + r(4 * N * -(-HW // 1024)) + 2 * r(4 * N * maxc)
        assert L.mr_db_contours_workspace_bytes(N, H, W, maxc) == want
    assert L.mr_db_contours_workspace_bytes(1, 1 << 14, 1 << 14, 10) == 0          # H * W >= 2^28
    assert L.mr_db_contours_workspace_bytes(1, (1 << 14) - 1, 1 << 14, 10) > 0
    assert L.mr_db_contours_workspace_bytes(1, 8, 8, -1) == 0
    fake = 0x10000                                     # never dereferenced: the checks come first
    call = lambda dest, N, H, W, maxc, ws, nbytes, pts, cap, off, cnt, tot: L.mr_db_contours_f32(  # noqa: E731
        dest, N, H, W, 0.3, maxc, ws, nbytes, pts, cap, off, cnt, tot, None)
    ok = int(L.mr_db_contours_workspace_bytes(2, 8, 8, 4))
    assert call(None, 0, 8, 8, 4, None, 0, None, 0, None, None, None) == 0          # empty batch: nothing to do
    assert call(fake, -1, 8, 8, 4, fake, ok, fake, 256, fake, fake, fake) == 4
    assert call(fake, 2, 0, 8, 4, fake, ok, fake, 256, fake, fake, fake) == 4
    assert call(fake, 2, 8, 8, -1, fake, ok, fake, 256, fake, fake, fake) == 4
    assert call(fake, 2, 8, 8, 4, fake, ok, fake, -1, fake, fake, fake) == 4
    assert call(fake, 1, 1 << 14, 1 << 14, 4, fake, 1 << 40, fake, 256, fake, fake, fake) == 4
    assert call(fake, 2, 8, 8, 4, fake, ok - 1, fake, 256, fake, fake, fake) == 4    # workspace too small
    assert call(None, 2, 8, 8, 4, fake, ok, fake, 256, fake, fake, fake) == 1
    assert call(fake, 2, 8, 8, 4, None, ok, fake, 256, fake, fake, fake) == 1
    assert call(fake, 2, 8, 8, 4, fake, ok, None, 256, fake, fake, fake) == 1
    assert call(fake, 2, 8, 8, 4, fake, ok, fake, 256, None, fake, fake) == 1
    assert call(fake, 2, 8, 8, 4, fake, ok, fake, 256, fake, None, fake) == 1
    assert call(fake, 2, 8, 8, 4, fake, ok, fake, 256, fake, fake, None) == 1
    assert L.mr_db_box_candidates_workspace_bytes(4, 1000, 4 * 576 * 1024) == r(4 * 4 * (6 * 4 * 576 * 1024 + 2 * 1000))
    mb = int(L.mr_db_box_candidates_workspace_bytes(2, 4, 256))
    cand = lambda N, maxc, cap, ws, nbytes, H=8, W=8, pts=fake, off=fake, cnt=fake, pred=fake, out=fake: (  # noqa: E731
        L.mr_db_box_candidates_f32(pts, cap, off, cnt, pred, N, H, W, maxc, ws, nbytes, out, out, out, None))
    assert cand(0, 4, 256, None, 0, pts=None, off=None, cnt=None, pred=None, out=None) == 0
    assert cand(-1, 4, 256, fake, mb) == 4 and cand(2, -1, 256, fake, mb) == 4 and cand(2, 4, -1, fake, mb) == 4
    assert cand(2, 4, 256, fake, mb, H=0) == 4 and cand(2, 4, 256, fake, mb, H=1 << 14, W=1 << 14) == 4
    assert cand(2, 4, 256, fake, mb - 1) == 4
    assert cand(2, 4, 256, None, mb) == 1 and cand(2, 4, 256, fake, mb, off=None) == 1 and cand(2, 4, 256, fake, mb, pred=None) == 1
    assert cand(2, 4, 256, fake, mb, cnt=None) == 1 and cand(2, 4, 256, fake, mb, out=None) == 1


def test_surface_refuses_cpu_tensors():
    import torch
    from megreader_b200 import db_boxes
    with pytest.raises(NotImplementedError):
        db_boxes.find_contours(torch.zeros(1, 1, 8, 8))
    with pytest.raises(NotImplementedError):
        db_boxes.box_candidates(torch.zeros(1, 1, 8, 8), torch.zeros(1, 256, 2, dtype=torch.int32),
                                torch.zeros(1, 5, dtype=torch.int32), torch.zeros(1, dtype=torch.int32))


# ---------------------------------------------------------------------------------------------------- unclip and rescale
def _rotated_boxes(seed, n):
    rng = np.random.RandomState(seed)
    for i in range(n):
        c = rng.uniform(-20, 700, 2)
        w, h = rng.uniform(3, 300, 2) if i % 3 else rng.uniform(3, 8, 2)
        a = rng.uniform(0, np.pi) if i % 4 else 0.0
        R = np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
        box = (c + (np.array([[-w, -h], [w, -h], [w, h], [-w, h]]) / 2) @ R.T).astype(np.float32)
        yield np.ascontiguousarray(box if i % 2 else box[::-1])


def _unclip(harness, box, cap=4096):
    d = ctypes.c_double()
    xy = np.zeros((cap, 2), np.int32)
    n = harness.host_unclip(_p(box), ctypes.byref(d), _p(xy), cap)
    return d.value, xy[:max(n, 0)]


def _point_polygon_distance(p, poly):
    best = np.inf
    for i in range(len(poly)):
        a, b = poly[i].astype(np.float64), poly[(i + 1) % len(poly)].astype(np.float64)
        ab = b - a
        t = 0.0 if not ab.any() else np.clip(np.dot(p - a, ab) / np.dot(ab, ab), 0, 1)
        best = min(best, np.linalg.norm(p - (a + t * ab)))
    return best


def test_unclip_core_equals_oracle_restatement(harness):
    """the device routine and oracle/db_boxes_port.py restate Clipper's round offset independently: same distance, same points"""
    from oracle.db_boxes_port import clipper_round_offset, ring_area_length
    for box in _rotated_boxes(1, 3000):
        d, got = _unclip(harness, box)
        area, length = ring_area_length(box)
        assert d == area * 1.5 / length
        assert got.tolist() == [list(p) for p in clipper_round_offset(box, d)], box.tolist()


def test_unclip_invariants(harness):
    """Not pinned against pyclipper, so pinned by what Clipper's round offset guarantees for a convex path: every vertex lies
    within distance +- 1 of the (integer) box, the result is convex up to the integer rounding, and it has Clipper's arc step
    count, steps = min(pi / acos(1 - y / d), pi d) per turn with y = min(0.25, d / 4)"""
    import math
    checked = 0
    for box in _rotated_boxes(2, 1500):
        q = box.astype(np.int64)                    # AddPath truncation
        e = [q[(i + 1) % 4] - q[i] for i in range(4)]
        cross = [e[i][0] * e[(i + 1) % 4][1] - e[i][1] * e[(i + 1) % 4][0] for i in range(4)]
        if not (all(c > 0 for c in cross) or all(c < 0 for c in cross)):
            continue                                # only strictly convex integer quads
        d, pts = _unclip(harness, box)
        assert d > 0 and len(pts) > 4
        for p in pts:
            assert abs(_point_polygon_distance(p.astype(np.float64), q) - d) <= 1.0, (box.tolist(), p.tolist(), d)
        hull = cv2.convexHull(pts.astype(np.int32)).reshape(-1, 2)
        assert all(_point_polygon_distance(p.astype(np.float64), hull) <= 1.0 for p in pts)
        y = min(0.25, d / 4)
        steps = min(math.pi / math.acos(1 - y / d), math.pi * d)
        assert abs(len(pts) - (steps + 4)) <= 4, (len(pts), steps)
        checked += 1
    assert checked > 1000


def test_unclip_distance_positive_for_candidates(harness):
    """delta <= 0 never occurs for a box that passes sside >= 3"""
    for bm in random_bitmaps(7, 500):
        for c in cv2_contours(bm):
            box, sside = get_mini_boxes(np.ascontiguousarray(c.reshape(-1, 2), np.int32))
            if sside >= 3:
                assert _unclip(harness, np.ascontiguousarray(box, np.float32))[0] > 0


def test_rescale_equals_numpy_float32(harness):
    """np.clip(np.round(box / width * dest), 0, dest) on a float32 box: float32 steps, round half to even"""
    harness.host_rescale.restype = ctypes.c_int
    rng = np.random.RandomState(4)
    vals = np.concatenate([rng.uniform(-30, 1100, 20000), np.arange(-4, 1030, 0.5)]).astype(np.float32)
    for size, dest in ((1024, 1024), (1024, 1280), (577, 300), (640, 641)):
        want = np.clip(np.round(vals / size * dest), 0, dest)
        got = np.array([harness.host_rescale(ctypes.c_float(v), size, dest) for v in vals])
        assert np.array_equal(got, want.astype(np.int64)), (size, dest)


def test_boxes_capi_argument_checks_without_gpu():
    from megreader_b200 import _lib
    L = _lib.lib()
    fake = 0x10000
    assert L.mr_db_boxes_workspace_bytes(4, 576, 1024, 1000) > 0
    assert L.mr_db_boxes_workspace_bytes(65536, 8, 8, 10) == 0 and L.mr_db_boxes_workspace_bytes(1, 1 << 14, 1 << 14, 10) == 0
    nb = int(L.mr_db_boxes_workspace_bytes(2, 8, 8, 4))
    f = lambda N, H=8, W=8, maxc=4, ws=fake, nbytes=nb, b=fake, d=fake, out=fake: L.mr_db_boxes_f32(  # noqa: E731
        b, d, N, H, W, 0.3, 0.7, maxc, None, ws, nbytes, out, out, out, None)
    assert f(0, b=None, d=None, ws=None, out=None) == 0
    assert f(-1) == 4 and f(65536) == 4 and f(2, H=0) == 4 and f(2, maxc=-1) == 4 and f(2, nbytes=nb - 1) == 4
    assert f(2, b=None) == 1 and f(2, d=None) == 1 and f(2, ws=None) == 1 and f(2, out=None) == 1
    assert L.mr_db_contours_f32(fake, 65536, 8, 8, 0.3, 4, fake, 1 << 40, fake, 256, fake, fake, fake, None) == 4
