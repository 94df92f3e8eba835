"""Seeded cases for the DB validation measure tests: gt quads (tests/db_targets_cases) with detections around them -- jittered
copies of gt boxes, noisy false positives, odd quads, rounded and clipped to int32 as the representer gives them -- and a
hand list of (gt, det) pairs at the edges of the evaluator: identical, contained, disjoint, edge- and corner-touching boxes,
axis-aligned integer boxes at IoU exactly 0.5 and one pixel either side, and intersection / area(det) exactly 0.5."""
import numpy as np

from tests.db_targets_cases import odd_quad, rotated_box


def _rect(x0, y0, x1, y1):
    return np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], np.float64)


def hand_pairs():
    """list of (name, gt [4, 2], det [4, 2]); names ending in '_exact_tie' have an exact IoU or precision of 0.5"""
    r = _rect
    cases = [
        ("identical", r(10, 10, 50, 30), r(10, 10, 50, 30)),
        ("contained", r(0, 0, 100, 100), r(20, 20, 40, 40)),
        ("containing", r(20, 20, 40, 40), r(0, 0, 100, 100)),
        ("disjoint", r(0, 0, 10, 10), r(20, 20, 30, 30)),
        ("edge_touch", r(0, 0, 10, 10), r(10, 0, 20, 10)),
        ("corner_touch", r(0, 0, 10, 10), r(10, 10, 20, 20)),
        ("two_thirds", r(0, 0, 30, 10), r(10, 0, 30, 10)),            # I = 200, U = 300
        ("iou_exact_tie", r(0, 0, 40, 10), r(0, 0, 20, 10)),          # I = 200, U = 400
        ("iou_exact_tie", r(0, 0, 30, 20), r(10, 0, 40, 20)),         # I = 400, U = 800
        ("iou_plus_px", r(0, 0, 40, 10), r(0, 0, 21, 10)),            # 210 / 400
        ("iou_minus_px", r(0, 0, 40, 10), r(0, 0, 19, 10)),           # 190 / 400
        ("iou_plus_px", r(0, 0, 30, 20), r(9, 0, 40, 20)),
        ("iou_minus_px", r(0, 0, 30, 20), r(11, 0, 40, 20)),
        ("precision_exact_tie", r(0, 0, 20, 10), r(10, 0, 30, 10)),  # I / area(det) = 100 / 200
        ("precision_exact_tie", r(0, 0, 100, 100), r(90, 0, 110, 50)),
        ("rotated_square", np.array([[50, 0], [100, 50], [50, 100], [0, 50]], np.float64), r(0, 0, 100, 100)),
        ("concave_dart", np.array([[0, 0], [50, 20], [100, 0], [50, 80]], np.float64), r(25, 0, 75, 40)),
        ("collinear_vertex", np.array([[0, 0], [10, 0], [20, 0], [20, 10]], np.float64), r(5, 0, 15, 5)),
        ("duplicate_corner", np.array([[0, 0], [0, 0], [20, 0], [0, 20]], np.float64), r(0, 0, 10, 10)),
        ("bow_tie", np.array([[0, 0], [10, 10], [10, 0], [0, 10]], np.float64), r(0, 0, 10, 10)),
        ("sliver_line", np.array([[0, 0], [5, 5], [10, 10], [0, 0]], np.float64), r(0, 0, 10, 10)),
    ]
    return cases


def jitter(rng, q, scale):
    return q + rng.normal(0, scale, q.shape)


def representer_box(q, H, W):
    """the representer's int32 box: rounded and clipped to the image"""
    b = np.round(q)
    b[:, 0] = np.clip(b[:, 0], 0, W)
    b[:, 1] = np.clip(b[:, 1], 0, H)
    return b.astype(np.int32)


def pair_corpus(rng, count, H=640, W=640):
    """count seeded (gt, det) float64 pairs of quads: mostly overlapping (jittered copies, shifted boxes), with odd quads
    (duplicates, slivers, concave, bow-ties, border-clipped integer corners) on either side and int32-rounded detections"""
    gts, dets = [], []
    for _ in range(count):
        g = odd_quad(rng, H, W) if rng.random() < 0.3 else rotated_box(rng, H, W)
        k = rng.integers(0, 5)
        if k == 0:
            d = jitter(rng, g, rng.uniform(0.5, 8))
        elif k == 1:
            d = representer_box(jitter(rng, g, rng.uniform(0.5, 5)), H, W).astype(np.float64)
        elif k == 2:
            d = odd_quad(rng, H, W)
            d = d - d.mean(0) + g.mean(0) + rng.normal(0, 10, 2)
        elif k == 3:                                 # axis-aligned integer boxes
            x0, y0 = rng.integers(0, 500, 2)
            g = _rect(x0, y0, x0 + rng.integers(1, 60), y0 + rng.integers(1, 40))
            d = g + rng.integers(-20, 21, 2)
            d[2:, :] += rng.integers(-10, 11, 2) * np.array([[1, 1], [0, 1]])
            d = _rect(d[:, 0].min(), d[:, 1].min(), d[:, 0].max(), d[:, 1].max())
        else:
            d = rotated_box(rng, H, W)
            d = d - d.mean(0) + g.mean(0) + rng.normal(0, 20, 2)
        gts.append(g)
        dets.append(d)
    return np.array(gts, np.float64), np.array(dets, np.float64)


def image_case(rng, H, W, n_gt, n_det, gt_dtype=np.float64, int_dets=True, noise=0.3, odd=0.2, dontcare=0.1):
    """one image: gt [n_gt, 4, 2] in gt_dtype, ignore tags, and n_det detections (int32 or float64 [n_det, 4, 2]) made of
    jittered gt boxes and, for the share `noise`, false positives and odd quads"""
    gt = np.array([odd_quad(rng, H, W) if rng.random() < odd else rotated_box(rng, H, W) for _ in range(n_gt)],
                  np.float64).reshape(n_gt, 4, 2)
    tags = rng.random(n_gt) < dontcare
    dets = []
    for _ in range(n_det):
        if n_gt and rng.random() > noise:
            dets.append(jitter(rng, gt[rng.integers(0, n_gt)], rng.uniform(0.5, 6)))
        elif rng.random() < 0.5:
            dets.append(rotated_box(rng, H, W, 4, 40))
        else:
            dets.append(odd_quad(rng, H, W))
    dets = np.array(dets, np.float64).reshape(n_det, 4, 2)
    if int_dets:
        dets = np.array([representer_box(d, H, W) for d in dets], np.int32).reshape(n_det, 4, 2)
    return gt.astype(gt_dtype), tags, dets


def batch_case(seed, N, H, W, gt_range, det_range, gt_dtype=np.float64, int_dets=True, **kw):
    rng = np.random.default_rng(seed)
    return [image_case(rng, H, W, int(rng.integers(gt_range[0], gt_range[1] + 1)), int(rng.integers(det_range[0], det_range[1] + 1)),
                       gt_dtype, int_dets, **kw) for _ in range(N)]
