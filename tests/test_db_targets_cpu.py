"""CPU: the PRODUCT's DB target routines (megreader_b200/csrc/db_targets_core.cuh -- the code the CUDA kernels of
csrc/db_targets.cu run) compiled for the host by tests/host_harness/db_targets_core_host.cpp, checked against
  * cv2.fillPoly on seeded int32 polygons of 3 to 200 vertices (arcs, self-intersecting, off the image, negative coordinates);
  * MakeBorderMap.distance (numpy, float64) bit for bit on grids through vertices, edge extensions and zero-length edges;
  * the invariants of Clipper's offset with its clean-up on seeded quads (distances to the quad, convexity, arc step counts)
    and the hand-computed shrink of a 100 x 40 box;
  * the oracle (oracle/db_targets_port.py) for whole images, bit for bit;
and the oracle against the reference's own MakeSegDetectionData / MakeBorderMap classes run on the oracle's shapely and
pyclipper restatements (skipped where the reference tree is absent)."""
import ctypes
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import db_targets_port as port
from tests.db_targets_cases import batch, odd_quad, rotated_box

cv2 = pytest.importorskip("cv2")

HERE = os.path.dirname(os.path.abspath(__file__))
SHRINK_K = 1 - np.power(0.4, 2)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("harness") / "libdb_targets_core_host.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                           "-I", os.path.join(HERE, "..", "megreader_b200", "csrc"),
                           os.path.join(HERE, "host_harness", "db_targets_core_host.cpp"), "-o", so])
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def host_targets(lib, polys, tags, H, W):
    polys = np.ascontiguousarray(polys.copy())
    n = len(polys)
    ign = np.ascontiguousarray(np.asarray(tags, dtype=np.uint8))
    out = {k: np.zeros((H, W), np.float32) for k in ("gt", "mask", "thresh_map", "thresh_mask")}
    status = np.zeros(n, np.int32)
    lib.host_make_targets(_p(polys), int(polys.dtype == np.float32), n, _p(ign), H, W, ctypes.c_double(SHRINK_K),
                          ctypes.c_double(8.0), ctypes.c_float(np.float32(0.7 - 0.3)), ctypes.c_float(0.3), _p(out["gt"]),
                          _p(out["mask"]), _p(out["thresh_map"]), _p(out["thresh_mask"]), _p(status))
    out.update(polygons=polys, ignore_tags=ign.astype(bool), status=status)
    return out


def raw_offset(lib, quad, delta):
    q = np.ascontiguousarray(quad, np.float64)
    xy = np.zeros((4096, 2), np.int32)
    n = lib.host_raw_offset(_p(q), ctypes.c_double(delta), _p(xy), 4096)
    assert n >= 0
    return xy[:n]


def clean(lib, path):
    path = np.ascontiguousarray(path, np.int32)
    out = np.zeros((4 * len(path) + 256, 2), np.int32)
    pieces = ctypes.c_int(0)
    m = lib.host_clean_offset(_p(path), len(path), _p(out), len(out), ctypes.byref(pieces))
    assert m >= 0
    return out[:m], pieces.value


# ---- cv2.fillPoly ----

def fill_polygons(rng, count):
    for _ in range(count):
        H, W = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        kind = rng.integers(0, 4)
        n = int(rng.integers(3, 201))
        if kind == 0:                                   # arc-like: points on a circle, possibly off the image
            c = rng.uniform(-0.5, 1.5, 2) * [W, H]
            r = rng.uniform(1, 1.5 * max(H, W))
            t = np.sort(rng.uniform(0, 2 * np.pi, n))
            pts = np.stack([c[0] + r * np.cos(t), c[1] + r * np.sin(t)], 1)
        elif kind == 1:                                 # self-intersecting scribble
            pts = rng.uniform(-0.5, 1.5, (n, 2)) * [W, H]
        elif kind == 2:                                 # few vertices, mostly inside
            n = int(rng.integers(3, 9))
            pts = rng.uniform(0, 1, (n, 2)) * [W, H]
        else:                                           # wholly or partly off the image, negative coordinates
            n = int(rng.integers(3, 30))
            pts = rng.uniform(-3, 1, (n, 2)) * [W, H]
        yield H, W, np.round(pts).astype(np.int32)


def test_fill_poly_matches_cv2(harness):
    rng = np.random.default_rng(7)
    count = 0
    for H, W, pts in fill_polygons(rng, 10000):
        want = np.zeros((H, W), np.uint8)
        cv2.fillPoly(want, [pts], 1)
        got = np.zeros((H, W), np.uint8)
        harness.host_fill_poly(_p(np.ascontiguousarray(pts)), len(pts), W, H, _p(got))
        assert np.array_equal(got, want), (H, W, pts.tolist())
        count += 1
    assert count == 10000


# ---- MakeBorderMap.distance ----

def test_edge_distance_bit_equal(harness):
    rng = np.random.default_rng(3)
    for k in range(300):
        dt = np.float32 if k % 2 else np.float64
        h, w = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        xs = np.broadcast_to(np.linspace(0, w - 1, num=w).reshape(1, w), (h, w))
        ys = np.broadcast_to(np.linspace(0, h - 1, num=h).reshape(h, 1), (h, w))
        a = np.array(rng.integers(-5, 45, 2), dt) if k % 3 else np.array(rng.uniform(-5, 45, 2), dt)
        b = a.copy() if k % 5 == 0 else np.array(rng.uniform(-5, 45, 2), dt)      # zero-length edges
        if k % 7 == 0:
            b = np.array([a[0], a[1] + rng.integers(1, 9)], dt)                      # through grid points
        with np.errstate(all="ignore"):
            want = port._distance(xs, ys, a, b)
        sd = np.square(a[0] - b[0]) + np.square(a[1] - b[1])
        got = np.zeros(h * w)
        X, Y = np.ascontiguousarray(xs.ravel()), np.ascontiguousarray(ys.ravel())
        harness.host_edge_distance(_p(X), _p(Y), h * w, *(ctypes.c_double(float(v)) for v in (a[0], a[1], b[0], b[1], sd)), _p(got))
        assert np.array_equal(got.view(np.uint64), want.ravel().view(np.uint64)) or \
            np.array_equal(np.isnan(got), np.isnan(want.ravel())) and np.array_equal(
                np.nan_to_num(got).view(np.uint64), np.nan_to_num(want.ravel()).view(np.uint64)), k


def test_edge_distance_equals_reference_method(harness):
    """the same, against MakeBorderMap.distance itself (skipped where the reference tree is absent)"""
    _, border = reference_processes()
    rng = np.random.default_rng(4)
    for k in range(60):
        dt = np.float32 if k % 2 else np.float64
        h, w = int(rng.integers(1, 30)), int(rng.integers(1, 30))
        xs = np.broadcast_to(np.linspace(0, w - 1, num=w).reshape(1, w), (h, w))
        ys = np.broadcast_to(np.linspace(0, h - 1, num=h).reshape(h, 1), (h, w))
        a = np.array(rng.integers(-3, 33, 2), dt)
        b = a.copy() if k % 4 == 0 else np.array(rng.uniform(-3, 33, 2), dt)
        with np.errstate(all="ignore"):
            want = border.distance(xs, ys, a, b).ravel()
        sd = np.square(a[0] - b[0]) + np.square(a[1] - b[1])
        got = np.zeros(h * w)
        X, Y = np.ascontiguousarray(xs.ravel()), np.ascontiguousarray(ys.ravel())
        harness.host_edge_distance(_p(X), _p(Y), h * w, *(ctypes.c_double(float(v)) for v in (a[0], a[1], b[0], b[1], sd)), _p(got))
        assert np.array_equal(np.isnan(got), np.isnan(want)), k
        assert np.array_equal(np.nan_to_num(got).view(np.uint64), np.nan_to_num(want).view(np.uint64)), k


# ---- the offset and its clean-up ----

def inside(p, quad, dist=False):
    """cv2.pointPolygonTest of the points p: +1 / 0 / -1 (inside / on / outside), or the signed distance when dist"""
    c = quad.astype(np.float32).reshape(-1, 1, 2)
    return np.array([cv2.pointPolygonTest(c, (float(x), float(y)), dist) for x, y in p])


def is_simple(q):
    def cross(a, b, c):
        return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
    for i, j in ((0, 2), (1, 3)):
        a, b, c, d = q[i], q[(i + 1) % 4], q[j], q[(j + 1) % 4]
        if cross(a, b, c) * cross(a, b, d) < 0 and cross(c, d, a) * cross(c, d, b) < 0:
            return False
    return True


def collinear_corners(q):
    """three distinct corners on one line (overlapping edges: the offset has no inside / outside there)"""
    pts = list(dict.fromkeys(tuple(p) for p in q))
    for i in range(len(pts)):
        a, b, c = pts[i - 2], pts[i - 1], pts[i]
        if (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0]) == 0:
            return True
    return False


def is_convex(q):
    m = len(q)
    z = []
    for i in range(m):
        a, b = q[(i + 1) % m] - q[i], q[(i + 2) % m] - q[(i + 1) % m]
        z.append(a[0] * b[1] - a[1] * b[0])
    return all(v >= 0 for v in z) or all(v <= 0 for v in z)


def arc_points(quad, delta):
    """Clipper's point count of the raw JT_ROUND offset of a convex quad padded by delta > 0 (corners truncated, distinct):
    per corner one point where |sin A * delta| < 1 and cos A > 0, else round(steps / 2 pi * |A|) (at least 1) arc steps plus
    the end point"""
    d = abs(delta)
    y = min(0.25, d * 0.25)
    steps = min(math.pi / math.acos(1 - y / d), d * math.pi)
    per_rad = steps / (2 * math.pi)
    q = [tuple(int(v) for v in p) for p in quad]
    if port.polygon_area(np.array(q, np.float64)) > 0:      # Clipper's positive orientation is the other way round
        q = q[::-1]
    normals = []                                    # GetUnitNormal(p[j], p[j + 1])
    for j in range(4):
        dx, dy = float(q[(j + 1) % 4][0] - q[j][0]), float(q[(j + 1) % 4][1] - q[j][1])
        f = 1.0 / math.sqrt(dx * dx + dy * dy)
        normals.append((dy * f, -(dx * f)))
    n = 0
    for j in range(4):
        (kx, ky), (jx, jy) = normals[j - 1], normals[j]
        sin_a, cos_a = kx * jy - jx * ky, kx * jx + jy * ky
        if abs(sin_a * delta) < 1 and cos_a > 0:
            n += 1
        else:
            n += max(port._round(per_rad * abs(math.atan2(min(max(sin_a, -1.0), 1.0), kx * jx + ky * jy))), 1) + 1
    return n


def test_clean_up_invariants(harness):
    rng = np.random.default_rng(11)
    H, W = 640, 640
    counts = dict(quads=0, convex_not_4=0, convex=0, shrink_checked=0, pad_checked=0, shrink_empty=0, pieces=0, steps=0)
    while counts["quads"] < 10000:
        q = odd_quad(rng, H, W) if rng.random() < 0.5 else rotated_box(rng, H, W)
        q[:, 0] = np.clip(q[:, 0], 0, W - 1)
        q[:, 1] = np.clip(q[:, 1], 0, H - 1)
        qi = np.trunc(q)
        if len({tuple(p) for p in qi}) < 3 or abs(port.polygon_area(qi)) < 1 or not is_simple(qi) or collinear_corners(qi):
            continue
        counts["quads"] += 1
        area, length = port.ring_area_length(q)
        d = area * SHRINK_K / length
        convex = is_convex(qi)
        counts["convex"] += convex
        shr, pieces = clean(harness, raw_offset(harness, q, -d))
        counts["pieces"] += pieces > 1
        if len(shr) == 0:
            counts["shrink_empty"] += 1
        else:
            # inside, at delta from the boundary up to the rounding of both coordinates
            sd = inside(shr, qi, True)
            assert (np.abs(sd - d) <= math.sqrt(2) + 1e-4).all(), (q.tolist(), d, shr.tolist())
            if convex:
                counts["convex_not_4"] += not (len(shr) <= 4 and is_convex(shr.astype(float)))
            counts["shrink_checked"] += 1
        raw = raw_offset(harness, q, d)
        pad, pieces = clean(harness, raw)
        assert len(pad) >= 3
        sd = inside(pad, qi, True)
        assert (np.abs(sd + d) <= math.sqrt(2) + 1e-4).all(), (q.tolist(), d, pad.tolist())
        if d > math.sqrt(2):
            assert (inside(qi, pad) > 0).all()
        counts["pad_checked"] += 1
        if convex and len({tuple(p) for p in qi}) == 4:
            assert len(raw) == arc_points(q, d)
            counts["steps"] += 1
    # a convex quad shrinks to the crossings of its four offset edges; where the quad is thinner than 2 delta next to a sharp
    # corner the spike edges of the raw path cut into that region and the rounded crossings add a vertex or a notch
    # (31 of 9,591 convex quads at this seed)
    assert counts["convex_not_4"] <= 0.01 * counts["convex"], counts
    assert counts["shrink_checked"] > 9000 and counts["steps"] > 3000, counts


def test_hand_case_box():
    box = np.array([[0, 0], [100, 0], [100, 40], [0, 40]], np.float64)
    area, length = port.ring_area_length(box)
    d = area * SHRINK_K / length
    assert d == 12.0
    off = port.PyclipperOffset()
    off.AddPath(box)
    (shr,) = off.Execute(-d)
    assert sorted(map(tuple, shr)) == [(12, 12), (12, 28), (88, 12), (88, 28)]


def test_hand_case_box_product(harness):
    box = np.array([[0, 0], [100, 0], [100, 40], [0, 40]], np.float64)
    shr, pieces = clean(harness, raw_offset(harness, box, -12.0))
    assert pieces == 1 and sorted(map(tuple, shr.tolist())) == [(12, 12), (12, 28), (88, 12), (88, 28)]


# ---- whole images ----

@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_host_targets_equal_oracle(harness, dtype):
    counted = np.zeros(8, int)
    for seed in range(6):
        for polys, tags in batch(100 + seed, 4, 320, 480, 0, 30, dtype, odd=0.5):
            want = port.make_targets(polys.copy(), tags, (320, 480))
            got = host_targets(harness, polys, tags, 320, 480)
            for k in ("mask", "thresh_map", "thresh_mask", "polygons", "ignore_tags", "status"):
                assert np.array_equal(got[k].view(np.uint8), np.ascontiguousarray(want[k]).view(np.uint8)), k
            assert np.array_equal(got["gt"], want["gt"][0])
            counted += [(want["status"] >> b & 1).sum() for b in range(8)]
    assert counted[1] and counted[2]              # |area| < 1 and sub-8 px text occur


# ---- the oracle against the reference's own classes ----

def reference_processes():
    from oracle import ref_loader
    if not ref_loader.install():
        pytest.skip("reference tree not present")
    import sys
    sys.modules["shapely.geometry"].Polygon = port.Polygon
    pc = sys.modules["pyclipper"]
    pc.PyclipperOffset, pc.JT_ROUND, pc.ET_CLOSEDPOLYGON = port.PyclipperOffset, port.JT_ROUND, port.ET_CLOSEDPOLYGON
    seg = ref_loader.load("data.processes.make_seg_detection_data").MakeSegDetectionData()
    border = ref_loader.load("data.processes.make_border_map").MakeBorderMap()
    return seg, border


def run_reference(seg, border, polys, tags, H, W):
    data = dict(image=np.zeros((H, W, 3), np.float32), polygons=polys.copy(), ignore_tags=[bool(t) for t in tags], filename="x")
    with np.errstate(all="ignore"):
        data = seg.process(data)
        data = border.process(data)
    return data


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_oracle_equals_reference_classes(dtype):
    seg, border = reference_processes()
    for polys, tags in batch(200, 6, 256, 384, 0, 25, dtype, odd=0.3):
        want = port.make_targets(polys.copy(), tags, (256, 384))
        if (want["status"] & port.PAD_EMPTY).any():
            continue                                # the reference raises IndexError there
        got = run_reference(seg, border, polys, tags, 256, 384)
        for k in ("gt", "mask", "thresh_map", "thresh_mask", "polygons"):
            assert np.array_equal(np.asarray(got[k]).view(np.uint8), np.ascontiguousarray(want[k]).view(np.uint8)), k
        assert list(map(bool, got["ignore_tags"])) == list(want["ignore_tags"])
