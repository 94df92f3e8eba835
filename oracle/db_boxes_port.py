"""CPU restatement of MegReader's SegDetectorRepresenter (structure/representers/seg_detector_representer.py:32-168) as it has to
run today, with exactly three environment fixes and nothing else changed:

  1. cv2.findContours returns two values under OpenCV 4 (the reference unpacks the OpenCV 3 triple);
  2. `int` for the removed `np.int`;
  3. pyclipper and shapely are not dependencies of this project: the unclip's Polygon(box).area / .length are the GEOS ring
     formulas in double, and PyclipperOffset(JT_ROUND, ET_CLOSEDPOLYGON).Execute(distance) is a Python restatement of the
     published Clipper 6.4.2 ClipperOffset (AddPath on the truncated corners, FixOrientations, DoOffset with DoRound,
     Round() half away from zero) WITHOUT its final ctUnion / pftPositive clean-up.  For the offset of a box the union gives
     the same region, so the second cv2.minAreaRect sees the same convex hull; the order of the points -- and with it which of
     several equal-area rectangles minAreaRect reports -- can differ.  This restatement is NOT pinned against pyclipper; the
     tests pin its invariants (vertices within distance +- 1 of the box, convex for convex boxes, Clipper's arc step count).

cv2 does the contours, minAreaRect, boxPoints, fillPoly and mean, as in the reference.  Debug drawing is not reproduced."""
import math

import cv2
import numpy as np


def ring_area_length(box):
    """GEOS Area::ofRing and Length::ofLine of the closed ring of the [4, 2] box (float64)"""
    x = [float(box[i % 4][0]) for i in range(5)]
    y = [float(box[i % 4][1]) for i in range(5)]
    s = 0.0
    for i in range(1, 4):
        s += (x[i] - x[0]) * (y[i - 1] - y[i + 1])
    length = 0.0
    for i in range(4):
        dx, dy = x[i + 1] - x[i], y[i + 1] - y[i]
        length += math.sqrt(dx * dx + dy * dy)
    return abs(s / 2.0), length


def _round(v):
    return int(v - 0.5) if v < 0 else int(v + 0.5)


def clipper_round_offset(box, delta, arc_tolerance=0.25):
    """ClipperOffset.Execute(delta) of one closed JT_ROUND path, before the union clean-up: list of (x, y) int points"""
    pts = [(int(p[0]), int(p[1])) for p in box]           # AddPath: cInt truncation
    hi = len(pts) - 1
    while hi > 0 and pts[0] == pts[hi]:
        hi -= 1
    path = [pts[0]]
    for p in pts[1:hi + 1]:
        if p != path[-1]:
            path.append(p)
    if len(path) < 3:
        return []
    area = 0.0
    j = len(path) - 1
    for i in range(len(path)):
        area += (float(path[j][0]) + path[i][0]) * (float(path[j][1]) - path[i][1])
        j = i
    if not (-area * 0.5 >= 0):                             # FixOrientations
        path.reverse()
    d = abs(delta)
    y = d * 0.25 if arc_tolerance > d * 0.25 else arc_tolerance
    steps = math.pi / math.acos(1 - y / d)
    if steps > d * math.pi:
        steps = d * math.pi
    s, c = math.sin(2 * math.pi / steps), math.cos(2 * math.pi / steps)
    per_rad = steps / (2 * math.pi)
    if delta < 0:
        s = -s
    n = len(path)
    normals = []
    for j in range(n):
        (x0, y0), (x1, y1) = path[j], path[(j + 1) % n]
        dx, dy = float(x1 - x0), float(y1 - y0)
        f = 1.0 / math.sqrt(dx * dx + dy * dy)
        normals.append((dy * f, -(dx * f)))
    out = []
    k = n - 1
    for j in range(n):
        (px, py), (kx, ky), (jx, jy) = path[j], normals[k], normals[j]
        sin_a = kx * jy - jx * ky
        joined = False
        if abs(sin_a * delta) < 1.0:
            if kx * jx + jy * ky > 0:
                out.append((_round(px + kx * delta), _round(py + ky * delta)))
                joined = True
        elif sin_a > 1.0:
            sin_a = 1.0
        elif sin_a < -1.0:
            sin_a = -1.0
        if not joined:
            if sin_a * delta < 0:
                out += [(_round(px + kx * delta), _round(py + ky * delta)), (px, py),
                        (_round(px + jx * delta), _round(py + jy * delta))]
            else:
                a = math.atan2(sin_a, kx * jx + ky * jy)
                st = max(_round(per_rad * abs(a)), 1)
                X, Y = kx, ky
                for _ in range(st):
                    out.append((_round(px + X * delta), _round(py + Y * delta)))
                    X, Y = X * c - s * Y, X * s + Y * c
                out.append((_round(px + jx * delta), _round(py + jy * delta)))
        k = j
    return out


class SegDetectorRepresenter:
    def __init__(self, thresh=0.3, box_thresh=0.7, max_candidates=100, resize=False, dest='binary'):
        self.thresh, self.box_thresh, self.max_candidates, self.resize, self.dest = thresh, box_thresh, max_candidates, resize, dest
        self.min_size = 3

    def represent(self, batch, _pred):
        pred = _pred[self.dest]
        segmentation = pred > self.thresh
        boxes_batch = []
        for batch_index in range(batch['image'].size(0)):
            height, width = batch['shape'][batch_index]
            boxes_batch.append(self.boxes_from_bitmap(_pred['binary'][batch_index], segmentation[batch_index], width, height))
        return boxes_batch, _pred

    def boxes_from_bitmap(self, pred, _bitmap, dest_width, dest_height):
        bitmap = _bitmap.data.cpu().numpy()[0]
        pred = pred.cpu().detach().numpy()[0]
        height, width = bitmap.shape
        boxes = []
        contours, _ = cv2.findContours((bitmap * 255).astype(np.uint8), cv2.RETR_LIST, cv2.CHAIN_APPROX_NONE)
        for contour in contours[:self.max_candidates]:
            points, sside = self.get_mini_boxes(contour)
            if sside < self.min_size:
                continue
            points = np.array(points)
            score = self.box_score_fast(pred, points.reshape(-1, 2))
            if self.box_thresh > score:
                continue
            box = self.unclip(points).reshape(-1, 1, 2)
            if len(box) == 0:                              # Clipper returns no path for a box of < 3 distinct points
                continue
            box, sside = self.get_mini_boxes(box)
            if sside < self.min_size + 2:
                continue
            box = np.array(box)
            if not self.resize:
                dest_width, dest_height = width, height
            box[:, 0] = np.clip(np.round(box[:, 0] / width * dest_width), 0, dest_width)
            box[:, 1] = np.clip(np.round(box[:, 1] / height * dest_height), 0, dest_height)
            boxes.append(box.tolist())
        return boxes

    def unclip(self, box):
        area, length = ring_area_length(box)
        return np.array(clipper_round_offset(box, area * 1.5 / length), dtype=np.int64)

    def get_mini_boxes(self, contour):
        bounding_box = cv2.minAreaRect(contour)
        points = sorted(list(cv2.boxPoints(bounding_box)), key=lambda x: x[0])
        index_1, index_4 = (0, 1) if points[1][1] > points[0][1] else (1, 0)
        index_2, index_3 = (2, 3) if points[3][1] > points[2][1] else (3, 2)
        return [points[index_1], points[index_2], points[index_3], points[index_4]], min(bounding_box[1])

    def box_score_fast(self, bitmap, _box):
        h, w = bitmap.shape[:2]
        box = _box.copy()
        xmin = np.clip(np.floor(box[:, 0].min()).astype(int), 0, w - 1)
        xmax = np.clip(np.ceil(box[:, 0].max()).astype(int), 0, w - 1)
        ymin = np.clip(np.floor(box[:, 1].min()).astype(int), 0, h - 1)
        ymax = np.clip(np.ceil(box[:, 1].max()).astype(int), 0, h - 1)
        mask = np.zeros((ymax - ymin + 1, xmax - xmin + 1), dtype=np.uint8)
        box[:, 0] = box[:, 0] - xmin
        box[:, 1] = box[:, 1] - ymin
        cv2.fillPoly(mask, box.reshape(1, -1, 2).astype(np.int32), 1)
        return cv2.mean(bitmap[ymin:ymax + 1, xmin:xmax + 1], mask)[0]
