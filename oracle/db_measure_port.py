"""CPU restatement of the DB detector's validation measure: QuadMeasurer (structure/measurers/quad_measurer.py) and
DetectionIoUEvaluator.evaluate_image / combine_results (concern/icdar2015_eval/detection/iou.py:13-206).

shapely is not a dependency of this project, so `Polygon` restates, for 4-point rings and in exact rational arithmetic
(fractions.Fraction), what the evaluator asks of it:
  * is_valid / is_simple: GEOS IsValidOp's rules for one ring -- finite coordinates; at least 3 distinct vertices once
    consecutive duplicates are dropped; no two non-adjacent edges sharing a point; no two adjacent edges overlapping beyond
    their shared vertex; nonzero area;
  * intersection(o).area: exact, by convex pieces and Sutherland-Hodgman clipping, rounded once to float;
  * union(o).area: area(a) + area(b) - intersection, exact, rounded once (equal to GEOS's overlay up to its rounding);
  * area and length: the GEOS ring formulas in double (ring_area_length), so the class can also stand in for
    db_targets_port.Polygon.
This is NOT pinned against shapely.  The evaluator and the measurer themselves are pinned: tests/test_db_measure_cpu.py
runs the reference's own iou.py and quad_measurer.py on this Polygon and requires equal results, and
oracle/make_db_measure_golden.py records them into tests/golden/db_measure_ref.npz.

Two deviations from the reference, both in DESIGN §7: where an image has no valid gt or no valid det, iouMat is [[0.0]]
(the reference's np.empty([1, 1]) is uninitialised), and measure() builds the detections per image, where the reference's
np.array(output[0]) raises on ragged batches under numpy >= 1.24."""
import math
from fractions import Fraction

import numpy as np



def ring_area_length(box):
    """GEOS Area::ofRing and Length::ofLine of the closed 4-point ring, in double (as oracle/db_boxes_port.py, restated here
    so that this module needs no cv2)"""
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


def _orient(a, b, c):
    v = (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
    return (v > 0) - (v < 0)


def _in_box(a, b, p):
    return min(a[0], b[0]) <= p[0] <= max(a[0], b[0]) and min(a[1], b[1]) <= p[1] <= max(a[1], b[1])


def _touch(a, b, c, d):
    o1, o2, o3, o4 = _orient(a, b, c), _orient(a, b, d), _orient(c, d, a), _orient(c, d, b)
    if o1 * o2 < 0 and o3 * o4 < 0:
        return True
    return ((o1 == 0 and _in_box(a, b, c)) or (o2 == 0 and _in_box(a, b, d)) or (o3 == 0 and _in_box(c, d, a))
            or (o4 == 0 and _in_box(c, d, b)))


def _twice_area(v):
    return sum(v[i][0] * v[(i + 1) % len(v)][1] - v[(i + 1) % len(v)][0] * v[i][1] for i in range(len(v)))


def _clip(subject, clip):
    """convex counter-clockwise subject clipped by the convex counter-clockwise clip polygon, exactly"""
    out = list(subject)
    m = len(clip)
    for e in range(m):
        if not out:
            break
        a, b = clip[e], clip[(e + 1) % m]
        side = lambda p: (b[0] - a[0]) * (p[1] - a[1]) - (b[1] - a[1]) * (p[0] - a[0])  # noqa: E731
        pts, out = out, []
        prev = pts[-1]
        sp = side(prev)
        for cur in pts:
            sc = side(cur)
            if (sp >= 0) != (sc >= 0):
                t = Fraction(sp) / (sp - sc)
                out.append((prev[0] + t * (cur[0] - prev[0]), prev[1] + t * (cur[1] - prev[1])))
            if sc >= 0:
                out.append(cur)
            prev, sp = cur, sc
    return out


def _box(v):
    xs, ys = [p[0] for p in v], [p[1] for p in v]
    return min(xs), min(ys), max(xs), max(ys)


def _overlap(a, b):
    return max(a[0], b[0]) < min(a[2], b[2]) and max(a[1], b[1]) < min(a[3], b[3])


class _Area:
    def __init__(self, area):
        self.area = area


class Polygon:
    """shapely.geometry.Polygon of a 4-point ring (see the module docstring)"""

    def __init__(self, points):
        pts = [(float(p[0]), float(p[1])) for p in points]
        if len(pts) != 4:
            raise ValueError("db_measure_port.Polygon: quads only, got %d points" % len(pts))
        self.points = pts
        self._valid = None
        self._ints = None
        self._exact = None

    @property
    def area(self):
        return ring_area_length(self.points)[0]

    @property
    def length(self):
        return ring_area_length(self.points)[1]

    def _distinct(self):
        v = []
        for p in self.points:
            if not v or p != v[-1]:
                v.append(p)
        while len(v) > 1 and v[-1] == v[0]:
            v.pop()
        return v

    def _scaled(self):
        """(e, the distinct vertices times 2^e as ints): every float is an integer over a power of two, so the exact
        arithmetic below runs on Python ints, with rationals only where Sutherland-Hodgman crosses an edge"""
        if self._ints is None:
            v = self._distinct()
            e = max(c.as_integer_ratio()[1].bit_length() - 1 for p in v for c in p)
            self._ints = (e, [tuple(int(Fraction(c) * 2 ** e) for c in p) for p in v])
        return self._ints

    @property
    def is_valid(self):
        if self._valid is None:
            self._valid = self._check()
        return self._valid

    is_simple = is_valid

    def _check(self):
        if not all(math.isfinite(c) for p in self.points for c in p):
            return False
        v = self._scaled()[1]
        m = len(v)
        if m < 3:
            return False
        for i in range(m):
            a, b, c = v[i - 1], v[i], v[(i + 1) % m]
            if _orient(a, b, c) == 0:
                ax, bx, cx = (a[0], b[0], c[0]) if a[0] != b[0] else (a[1], b[1], c[1])
                if (ax > bx) == (cx > bx):
                    return False                    # the two edges fold back over each other
        if m == 4 and (_touch(v[0], v[1], v[2], v[3]) or _touch(v[1], v[2], v[3], v[0])):
            return False
        return _twice_area(v) != 0

    def _pieces(self):
        """(e, convex pieces counter-clockwise in ints times 2^e with their boxes, twice the area times 4^e)"""
        if self._exact is None:
            e, v = self._scaled()
            s = _twice_area(v)
            if s < 0:
                v = v[::-1]
            reflex = [i for i in range(len(v)) if _orient(v[i - 1], v[i], v[(i + 1) % len(v)]) < 0]
            if not reflex:
                pieces = [v]
            else:
                r = reflex[0]
                w = v[r:] + v[:r]
                pieces = [[w[0], w[1], w[2]], [w[0], w[2], w[3]]]
            self._exact = (e, pieces, abs(s))
        return self._exact

    def exact_area(self):
        e, _, s2 = self._pieces()
        return Fraction(s2, 2 * 4 ** e)

    def exact_intersection(self, other):
        if not _overlap(_box(self.points), _box(other.points)):
            return Fraction(0)
        ea, pa, _ = self._pieces()
        eb, pb, _ = other._pieces()
        e = max(ea, eb)
        pa = [[(x << (e - ea), y << (e - ea)) for x, y in p] for p in pa]
        pb = [[(x << (e - eb), y << (e - eb)) for x, y in p] for p in pb]
        total = 0
        for a in pa:
            ba = _box(a)
            for b in pb:
                if _overlap(ba, _box(b)):
                    c = _clip(a, b)
                    if len(c) >= 3:
                        total += _twice_area(c)
        return Fraction(total) / (2 * 4 ** e)

    def intersection(self, other):
        return _Area(float(self.exact_intersection(other)))

    def union(self, other):
        return _Area(float(self.exact_area() + other.exact_area() - self.exact_intersection(other)))


# ---- the evaluator, restated ----

def evaluate_image(gt, pred, iou_constraint=0.5, area_precision_constraint=0.5):
    """DetectionIoUEvaluator.evaluate_image: gt a list of dict(points, ignore), pred a list of dict(points)"""
    gt_pols, gt_points, gt_dc = [], [], []
    for g in gt:
        if Polygon(g['points']).is_valid:
            gt_pols.append(Polygon(g['points']))
            gt_points.append(g['points'])
            if g['ignore']:
                gt_dc.append(len(gt_pols) - 1)
    log = "GT polygons: " + str(len(gt_pols)) + (" (" + str(len(gt_dc)) + " don't care)\n" if gt_dc else "\n")
    det_pols, det_points, det_dc = [], [], []
    for d in pred:
        pd = Polygon(d['points'])
        if not pd.is_valid:
            continue
        det_pols.append(pd)
        det_points.append(d['points'])
        for k in gt_dc:
            inter = float(gt_pols[k].exact_intersection(pd))
            area = pd.area
            if (0 if area == 0 else inter / area) > area_precision_constraint:
                det_dc.append(len(det_pols) - 1)
                break
    log += "DET polygons: " + str(len(det_pols)) + (" (" + str(len(det_dc)) + " don't care)\n" if det_dc else "\n")
    pairs = []
    iou_mat = [[0.0]]
    matched = 0
    if gt_pols and det_pols:
        iou = np.zeros((len(gt_pols), len(det_pols)))
        for i, pg in enumerate(gt_pols):
            for j, pd in enumerate(det_pols):
                inter = pd.exact_intersection(pg)
                if inter:
                    iou[i, j] = float(inter) / pd.union(pg).area
        det_taken = np.zeros(len(det_pols), bool)
        gt_dc_set, det_dc_set = set(gt_dc), set(det_dc)
        for i in range(len(gt_pols)):
            if i in gt_dc_set:
                continue
            for j in range(len(det_pols)):
                if not det_taken[j] and j not in det_dc_set and iou[i, j] > iou_constraint:
                    det_taken[j] = True
                    matched += 1
                    pairs.append({'gt': i, 'det': j})
                    log += "Match GT #" + str(i) + " with Det #" + str(j) + "\n"
                    break
        iou_mat = iou.tolist()
    gt_care = len(gt_pols) - len(gt_dc)
    det_care = len(det_pols) - len(det_dc)
    if gt_care == 0:
        recall = float(1)
        precision = float(0) if det_care > 0 else float(1)
    else:
        recall = float(matched) / gt_care
        precision = 0 if det_care == 0 else float(matched) / det_care
    hmean = 0 if (precision + recall) == 0 else 2.0 * precision * recall / (precision + recall)
    return {'precision': precision, 'recall': recall, 'hmean': hmean, 'pairs': pairs,
            'iouMat': [] if len(det_pols) > 100 else iou_mat, 'gtPolPoints': gt_points, 'detPolPoints': det_points,
            'gtCare': gt_care, 'detCare': det_care, 'gtDontCare': gt_dc, 'detDontCare': det_dc, 'detMatched': matched,
            'evaluationLog': log}


def combine_results(results):
    gt = sum(r['gtCare'] for r in results)
    det = sum(r['detCare'] for r in results)
    matched = sum(r['detMatched'] for r in results)
    recall = 0 if gt == 0 else float(matched) / gt
    precision = 0 if det == 0 else float(matched) / det
    hmean = 0 if recall + precision == 0 else 2 * recall * precision / (recall + precision)
    return {'precision': precision, 'recall': recall, 'hmean': hmean}


class AverageMeter:
    def __init__(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count
        return self


class QuadMeasurer:
    """QuadMeasurer with the restated evaluator; output[0] holds per image a list (or array) of [4, 2] boxes"""

    def measure(self, batch, output):
        results = []
        for polygons, pred, tags in zip(batch['polygons'], output[0], batch['ignore_tags']):
            pred = np.array(pred)
            gt = [dict(points=polygons[i], ignore=tags[i]) for i in range(len(polygons))]
            results.append(evaluate_image(gt, [dict(points=pred[i]) for i in range(len(pred))]))
        return results

    def validate_measure(self, batch, output):
        return self.measure(batch, output), [0]

    def gather_measure(self, raw_metrics, logger=None):
        raw_metrics = [m for batch_metrics in raw_metrics for m in batch_metrics]
        result = combine_results(raw_metrics)
        precision, recall, fmeasure = AverageMeter(), AverageMeter(), AverageMeter()
        precision.update(result['precision'], n=len(raw_metrics))
        recall.update(result['recall'], n=len(raw_metrics))
        fmeasure.update(2 * precision.val * recall.val / (precision.val + recall.val + 1e-8))
        return {'precision': precision, 'recall': recall, 'fmeasure': fmeasure}
