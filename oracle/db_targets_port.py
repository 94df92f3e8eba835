"""CPU restatement of the DB detector's two target processes, MakeSegDetectionData (data/processes/make_seg_detection_data.py:
21-100) and MakeBorderMap (make_border_map.py:24-121), with the same numpy and cv2 calls in the same order.

shapely and pyclipper are not dependencies of this project, so the two calls into them are restated:
  * Polygon(p).area / .length: the GEOS ring formulas in double (db_boxes_port.ring_area_length);
  * PyclipperOffset().AddPath(p, JT_ROUND, ET_CLOSEDPOLYGON).Execute(delta): db_boxes_port.clipper_round_offset for the raw
    offset path, then Execute's clean-up restated as the boundary of {winding of the raw path >= 1} (clean_offset below, the
    same rules as megreader_b200/csrc/db_targets_core.cuh).  When that region has several loops, Execute returns the one of
    largest |area| first (the first traced on ties); the reference uses element [0].
This restatement is NOT pinned against pyclipper; tests pin its invariants.

`Polygon` and `PyclipperOffset` have the shapes of the shapely / pyclipper names the reference uses, so the reference's own
classes can run on them (tests/test_db_targets_cpu.py, oracle/make_db_targets_golden.py).  Where the reference raises
IndexError (a pad with no polygon), draw_border_map here skips the polygon and counts it."""
import math

import cv2
import numpy as np

from oracle.db_boxes_port import _round, clipper_round_offset, ring_area_length

# per-polygon status bits, as the C-ABI reports them
IGNORED_IN, TINY_AREA, SMALL_TEXT, SHRINK_EMPTY, SHRINK_PIECES, PAD_EMPTY, PAD_PIECES, OVERFLOW = 1, 2, 4, 8, 16, 32, 64, 128

HORIZONTAL = -1.0E+40


def _cedge(x0, y0, x1, y1):
    bx, by, tx, ty = (x0, y0, x1, y1) if y0 >= y1 else (x1, y1, x0, y0)
    dx = HORIZONTAL if by == ty else float(tx - bx) / float(ty - by)
    return bx, by, tx, ty, dx


def _top_x(e, y):
    bx, by, tx, ty, dx = e
    return tx if y == ty else bx + _round(dx * float(y - by))


def clipper_intersect(e1, e2):
    """Clipper 6.4.2 IntersectPoint of two crossing edges (e1 the one of lower index), with ProcessHorizontal's point for a
    horizontal edge and the scan-beam clamps taken at the edges' common Y range"""
    h1, h2 = e1[4] == HORIZONTAL, e2[4] == HORIZONTAL
    if h1 or h2:
        Y = e1[1] if h1 else e2[1]
        return _top_x(e2 if h1 else e1, Y), Y
    if e1[4] == 0.0:
        X = e1[0]
        b2 = float(e2[1]) - float(e2[0]) / e2[4]
        Y = _round(float(X) / e2[4] + b2)
    elif e2[4] == 0.0:
        X = e2[0]
        b1 = float(e1[1]) - float(e1[0]) / e1[4]
        Y = _round(float(X) / e1[4] + b1)
    else:
        b1 = float(e1[0]) - float(e1[1]) * e1[4]
        b2 = float(e2[0]) - float(e2[1]) * e2[4]
        q = (b2 - b1) / (e1[4] - e2[4])
        Y = _round(q)
        X = _round(e1[4] * q + b1) if abs(e1[4]) < abs(e2[4]) else _round(e2[4] * q + b2)
    if Y < e1[3] or Y < e2[3]:
        Y = e1[3] if e1[3] > e2[3] else e2[3]
        X = _top_x(e1, Y) if abs(e1[4]) < abs(e2[4]) else _top_x(e2, Y)
    bot = min(e1[1], e2[1])
    if Y > bot:
        Y = bot
        X = _top_x(e2, Y) if abs(e1[4]) > abs(e2[4]) else _top_x(e1, Y)
    return X, Y


def _cross(a, b, c):
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def _sgn(v):
    return (v > 0) - (v < 0)


def _turn_class(cr, dt):
    return 0 if cr < 0 else 2 if cr > 0 else 1 if dt > 0 else 3


def _turns_left_of(cr, dt, cr2, dt2):
    a, b = _turn_class(cr, dt), _turn_class(cr2, dt2)
    if a != b:
        return a > b
    if a == 2:
        return dt * cr2 < dt2 * cr
    if a == 0:
        return dt * -cr2 > dt2 * -cr
    return False


def _clean_loop(loop):
    loop = list(loop)
    changed = True
    while changed and len(loop) >= 3:
        changed = False
        i = 0
        while i < len(loop) and len(loop) >= 3:
            m = len(loop)
            if _cross(loop[i - 1], loop[i], loop[(i + 1) % m]) == 0:
                del loop[i]
                changed = True
            else:
                i += 1
    if len(loop) < 3:
        return [], 0
    a = 0
    for i in range(len(loop)):
        (xj, yj), (xi, yi) = loop[i - 1], loop[i]
        a += xj * yi - xi * yj
    return loop, abs(a)


def clean_offset(path):
    """Execute's clean-up of the raw offset path (list of (x, y) ints): the loops bounding {winding >= 1}, the one of largest
    |area| first (first traced on ties), then the others in traced order"""
    n = len(path)
    if n < 3:
        return []
    P = path
    cr = []                                                # (edge, t, x, y) per crossing end
    for i in range(n):
        i1 = (i + 1) % n
        for j in range(i + 2, n):
            j1 = (j + 1) % n
            if j1 == i:
                continue
            d1 = _cross(P[i], P[i1], P[j])
            d2 = _cross(P[i], P[i1], P[j1])
            d3 = _cross(P[j], P[j1], P[i])
            d4 = _cross(P[j], P[j1], P[i1])
            if _sgn(d1) * _sgn(d2) >= 0 or _sgn(d3) * _sgn(d4) >= 0:
                continue
            X, Y = clipper_intersect(_cedge(*P[i], *P[i1]), _cedge(*P[j], *P[j1]))
            cr.append((i, float(d3) / float(d3 - d4), X, Y))
            cr.append((j, float(d1) / float(d1 - d2), X, Y))
    for i in range(n):                                     # raw vertices inside another edge
        i1 = (i + 1) % n
        ex, ey = P[i1][0] - P[i][0], P[i1][1] - P[i][1]
        len2 = ex * ex + ey * ey
        for v in range(n):
            if _cross(P[i], P[i1], P[v]) != 0:
                continue
            dot = (P[v][0] - P[i][0]) * ex + (P[v][1] - P[i][1]) * ey
            if 0 < dot < len2:
                cr.append((i, float(dot) / float(len2), P[v][0], P[v][1]))
    pieces = []
    for i in range(n):
        i1 = (i + 1) % n
        ends = sorted((t, k) for k, (e, t, _, _) in enumerate(cr) if e == i)
        a, ta = P[i], 0.0
        for t, k in ends + [(1.0, None)]:
            b = P[i1] if k is None else (cr[k][2], cr[k][3])
            if a != b:
                tm = (ta + t) * 0.5
                mx = float(P[i][0]) + tm * float(P[i1][0] - P[i][0])
                my = float(P[i][1]) + tm * float(P[i1][1] - P[i][1])
                th = 0.0
                for j in range(n):
                    if j == i:
                        continue
                    j1 = (j + 1) % n
                    ux, uy = float(P[j][0]) - mx, float(P[j][1]) - my
                    vx, vy = float(P[j1][0]) - mx, float(P[j1][1]) - my
                    th += math.atan2(ux * vy - uy * vx, ux * vx + uy * vy)
                if math.floor((th + math.pi) / (2 * math.pi) + 0.5) == 1.0:
                    pieces.append((a, b))
            a, ta = b, t
    used = [False] * len(pieces)
    loops = []
    for st in range(len(pieces)):
        if used[st]:
            continue
        loop, cur = [], st
        while cur is not None:
            used[cur] = True
            (a, b) = pieces[cur]
            loop.append(a)
            ux, uy = b[0] - a[0], b[1] - a[1]
            nxt, ncr, ndt = None, 0, 0
            for k, (c, d) in enumerate(pieces):
                if used[k] or c != b:
                    continue
                vx, vy = d[0] - c[0], d[1] - c[1]
                crs, dt = ux * vy - uy * vx, ux * vx + uy * vy
                if nxt is None or _turns_left_of(crs, dt, ncr, ndt):
                    nxt, ncr, ndt = k, crs, dt
            cur = nxt
        loop, area2 = _clean_loop(loop)
        if loop:
            loops.append((area2, loop))
    if not loops:
        return []
    best = 0
    for k in range(1, len(loops)):
        if loops[k][0] > loops[best][0]:
            best = k
    return [loops[best][1]] + [lp for k, (_, lp) in enumerate(loops) if k != best]


class Polygon:
    """shapely.geometry.Polygon of a [4, 2] ring: .area and .length (GEOS ring formulas in double)"""

    def __init__(self, points):
        self.area, self.length = ring_area_length(np.asarray(points))


class PyclipperOffset:
    """pyclipper.PyclipperOffset for one closed JT_ROUND path (arc tolerance 0.25).  `pieces` of the last Execute is the
    number of loops of the cleaned result."""
    pieces = 0

    def __init__(self):
        self.path = None

    def AddPath(self, path, join_type=None, end_type=None):
        self.path = [tuple(p) for p in path]

    def Execute(self, delta):
        out = clean_offset(clipper_round_offset(self.path, delta))
        self.pieces = len(out)
        return [[list(p) for p in lp] for lp in out]


JT_ROUND, ET_CLOSEDPOLYGON = 2, 3        # pyclipper's values; the restatement knows only these


def polygon_area(polygon):
    edge = [(polygon[(i + 1) % 4][0] - polygon[i][0]) * (polygon[(i + 1) % 4][1] + polygon[i][1]) for i in range(4)]
    return np.sum(edge) / 2.


def validate_polygons(polygons, ignore_tags, h, w, status=None):
    """validate_polygons in the polygons' dtype, in place: clip, |area| < 1 -> ignore, area > 0 -> (0, 3, 2, 1)"""
    if polygons.shape[0] == 0:
        return polygons, ignore_tags
    polygons[:, :, 0] = np.clip(polygons[:, :, 0], 0, w - 1)
    polygons[:, :, 1] = np.clip(polygons[:, :, 1], 0, h - 1)
    for i in range(polygons.shape[0]):
        area = polygon_area(polygons[i])
        if abs(area) < 1:
            ignore_tags[i] = True
            if status is not None:
                status[i] |= TINY_AREA
        if area > 0:
            polygons[i] = polygons[i][(0, 3, 2, 1), :]
    return polygons, ignore_tags


def _shrink_distance(polygon, shrink_ratio):
    shape = Polygon(polygon)
    return shape.area * (1 - np.power(shrink_ratio, 2)) / shape.length


def seg_detection_data(polygons, ignore_tags, h, w, min_text_size=8, shrink_ratio=0.4, status=None):
    """MakeSegDetectionData.process: -> (gt [1, h, w], mask [h, w], polygons, ignore_tags); status (a list) gets the bits"""
    polygons, ignore_tags = validate_polygons(polygons, ignore_tags, h, w, status)
    gt = np.zeros((1, h, w), dtype=np.float32)
    mask = np.ones((h, w), dtype=np.float32)
    for i in range(polygons.shape[0]):
        polygon = polygons[i]
        height = min(np.linalg.norm(polygon[0] - polygon[3]), np.linalg.norm(polygon[1] - polygon[2]))
        width = min(np.linalg.norm(polygon[0] - polygon[1]), np.linalg.norm(polygon[2] - polygon[3]))
        if status is not None and min(height, width) < min_text_size and not (status[i] & (IGNORED_IN | TINY_AREA)):
            status[i] |= SMALL_TEXT
        if ignore_tags[i] or min(height, width) < min_text_size:
            cv2.fillPoly(mask, polygon.astype(np.int32)[np.newaxis, :, :], 0)
            ignore_tags[i] = True
            continue
        distance = _shrink_distance(polygon, shrink_ratio)
        offset = PyclipperOffset()
        offset.AddPath([tuple(p) for p in polygon], JT_ROUND, ET_CLOSEDPOLYGON)
        shrinked = offset.Execute(-distance)
        if shrinked == []:
            cv2.fillPoly(mask, polygon.astype(np.int32)[np.newaxis, :, :], 0)
            ignore_tags[i] = True
            if status is not None:
                status[i] |= SHRINK_EMPTY
            continue
        if status is not None and offset.pieces > 1:
            status[i] |= SHRINK_PIECES
        cv2.fillPoly(gt[0], [np.array(shrinked[0]).reshape(-1, 2).astype(np.int32)], 1)
    return gt, mask, polygons, ignore_tags


def _distance(xs, ys, point_1, point_2):
    square_distance_1 = np.square(xs - point_1[0]) + np.square(ys - point_1[1])
    square_distance_2 = np.square(xs - point_2[0]) + np.square(ys - point_2[1])
    square_distance = np.square(point_1[0] - point_2[0]) + np.square(point_1[1] - point_2[1])
    cosin = (square_distance - square_distance_1 - square_distance_2) / (2 * np.sqrt(square_distance_1 * square_distance_2))
    square_sin = np.nan_to_num(1 - np.square(cosin))
    result = np.sqrt(square_distance_1 * square_distance_2 * square_sin / square_distance)
    result[cosin < 0] = np.sqrt(np.fmin(square_distance_1, square_distance_2))[cosin < 0]
    return result


def draw_border_map(polygon, canvas, mask, shrink_ratio=0.4):
    """MakeBorderMap.draw_border_map; returns the status bits of the pad (PAD_EMPTY: nothing drawn)"""
    polygon = np.array(polygon)
    distance = _shrink_distance(polygon, shrink_ratio)
    offset = PyclipperOffset()
    offset.AddPath([tuple(p) for p in polygon], JT_ROUND, ET_CLOSEDPOLYGON)
    padded = offset.Execute(distance)
    if not padded:
        return PAD_EMPTY
    padded_polygon = np.array(padded[0])
    cv2.fillPoly(mask, [padded_polygon.astype(np.int32)], 1.0)
    xmin, xmax = padded_polygon[:, 0].min(), padded_polygon[:, 0].max()
    ymin, ymax = padded_polygon[:, 1].min(), padded_polygon[:, 1].max()
    width, height = xmax - xmin + 1, ymax - ymin + 1
    polygon[:, 0] = polygon[:, 0] - xmin
    polygon[:, 1] = polygon[:, 1] - ymin
    xs = np.broadcast_to(np.linspace(0, width - 1, num=width).reshape(1, width), (height, width))
    ys = np.broadcast_to(np.linspace(0, height - 1, num=height).reshape(height, 1), (height, width))
    distance_map = np.zeros((polygon.shape[0], height, width), dtype=np.float32)
    for i in range(polygon.shape[0]):
        j = (i + 1) % polygon.shape[0]
        distance_map[i] = np.clip(_distance(xs, ys, polygon[i], polygon[j]) / distance, 0, 1)
    distance_map = distance_map.min(axis=0)
    x0, x1 = min(max(0, xmin), canvas.shape[1] - 1), min(max(0, xmax), canvas.shape[1] - 1)
    y0, y1 = min(max(0, ymin), canvas.shape[0] - 1), min(max(0, ymax), canvas.shape[0] - 1)
    canvas[y0:y1 + 1, x0:x1 + 1] = np.fmax(1 - distance_map[y0 - ymin:y1 - ymax + height, x0 - xmin:x1 - xmax + width],
                                           canvas[y0:y1 + 1, x0:x1 + 1])
    return PAD_PIECES if offset.pieces > 1 else 0


def border_map(polygons, ignore_tags, h, w, shrink_ratio=0.4, thresh_min=0.3, thresh_max=0.7, status=None):
    """MakeBorderMap.process: -> (thresh_map [h, w], thresh_mask [h, w])"""
    canvas = np.zeros((h, w), dtype=np.float32)
    mask = np.zeros((h, w), dtype=np.float32)
    for i in range(polygons.shape[0]):
        if ignore_tags[i]:
            continue
        bits = draw_border_map(polygons[i], canvas, mask, shrink_ratio)
        if status is not None:
            status[i] |= bits
    canvas = canvas * (thresh_max - thresh_min) + thresh_min
    return canvas, mask


def make_targets(polygons, ignore_tags, size, shrink_ratio=0.4, min_text_size=8, thresh_min=0.3, thresh_max=0.7):
    """Both processes for one image: polygons [n, 4, 2] float32/float64 and ignore_tags [n] (copied), size (H, W) ->
    dict(gt, mask, thresh_map, thresh_mask, polygons, ignore_tags, status) as the device call returns them"""
    h, w = size
    polygons = np.array(polygons).reshape(-1, 4, 2)
    ignore = [bool(t) for t in ignore_tags]
    status = [IGNORED_IN if t else 0 for t in ignore]
    with np.errstate(all="ignore"):
        gt, mask, polygons, ignore = seg_detection_data(polygons, ignore, h, w, min_text_size, shrink_ratio, status)
        thresh_map, thresh_mask = border_map(polygons, ignore, h, w, shrink_ratio, thresh_min, thresh_max, status)
    return dict(gt=gt, mask=mask, thresh_map=thresh_map, thresh_mask=thresh_mask, polygons=polygons,
                ignore_tags=np.array(ignore, dtype=bool).reshape(-1), status=np.array(status, dtype=np.int32).reshape(-1))
