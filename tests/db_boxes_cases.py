"""Seeded inputs of the DB contour step (megreader_b200/db_boxes.py), numpy only so that the GPU tests can rebuild them where cv2 or
scipy are missing:

    random_bitmaps(seed, n)     small noisy bitmaps (3..40 px a side), some opened or closed
    adversarial_bitmaps()       one-pixel lines and rings, diagonal-only contacts, nested holes / islands, frame cases, ...
    prob_maps(seed, N, H, W)    DB-like probability maps: the text boxes of tests/db_data.db_batch, blurred, through a sigmoid,
                                plus noise -- hundreds of contours per image, small, broken and holed ones included
and the reference contour list (cv2.findContours(RETR_LIST, CHAIN_APPROX_NONE), as seg_detector_representer.py:73-75 calls it)
in the digest form of tests/golden/db_contours_ref.npz."""
import hashlib

import numpy as np

from tests.db_data import db_batch


def _open_close(bm, close):
    H, W = bm.shape
    p = np.pad(bm, 1, constant_values=0)
    win = lambda a, f: f([a[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)], axis=0)  # noqa: E731
    if close:
        d = win(p, np.max)
        return win(np.pad(d, 1, constant_values=1), np.min).astype(np.uint8)
    e = win(p, np.min)
    return win(np.pad(e, 1, constant_values=0), np.max).astype(np.uint8)


def random_bitmaps(seed, n):
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        H, W = rng.randint(3, 41, 2)
        bm = (rng.rand(H, W) < rng.uniform(0.2, 0.8)).astype(np.uint8)
        k = rng.randint(4)
        if k == 1:
            bm = _open_close(bm, False)
        elif k == 2:
            bm = _open_close(bm, True)
        out.append(bm)
    return out


def adversarial_bitmaps():
    cases = {}
    z = lambda h, w: np.zeros((h, w), np.uint8)  # noqa: E731
    cases["empty"] = z(7, 9)
    cases["full"] = np.ones((7, 9), np.uint8)
    cases["one_pixel_map"] = np.ones((1, 1), np.uint8)
    cases["one_row"] = (np.arange(13) % 3 != 0).astype(np.uint8)[None]
    cases["one_column"] = (np.arange(11) % 4 != 1).astype(np.uint8)[:, None]
    a = z(9, 9); a[4, 4] = 1; cases["single_pixel"] = a
    a = z(9, 12); a[0, 0] = a[8, 11] = a[0, 11] = a[8, 0] = 1; cases["corner_pixels"] = a
    a = z(5, 12); a[2, 1:11] = 1; cases["horizontal_line"] = a
    a = z(12, 5); a[1:11, 2] = 1; cases["vertical_line"] = a
    a = z(12, 12); np.fill_diagonal(a, 1); cases["diagonal_line"] = a
    a = z(12, 12); np.fill_diagonal(a[:, ::-1], 1); cases["anti_diagonal_line"] = a
    a = z(9, 9); a[1, 1:8] = a[7, 1:8] = a[1:8, 1] = a[1:8, 7] = 1; cases["one_pixel_ring"] = a
    a = z(9, 9)
    for y, x in ((1, 4), (2, 3), (3, 2), (4, 1), (5, 2), (6, 3), (7, 4), (6, 5), (5, 6), (4, 7), (3, 6), (2, 5)):
        a[y, x] = 1
    cases["diagonal_ring"] = a                        # 8-connected ring around a hole that is open diagonally only
    a = z(6, 6); a[1, 1] = a[2, 2] = a[1, 3] = a[3, 1] = 1; cases["diagonal_contacts"] = a
    cases["checkerboard"] = (np.indices((16, 18)).sum(0) % 2).astype(np.uint8)
    a = z(15, 15)
    a[1:14, 1:14] = 1; a[3:12, 3:12] = 0; a[5:10, 5:10] = 1; a[7, 7] = 0
    cases["nested_holes_and_islands"] = a
    a = np.ones((8, 10), np.uint8); a[0, 3:6] = 0; a[3:5, 0] = 0; a[7, 8] = 0; a[3, 4:6] = 0
    cases["frame_holes"] = a                          # background touching the frame is no hole; the inner one is
    a = np.ones((7, 7), np.uint8); a[1::2, 1::2] = 0; cases["grid_of_holes"] = a
    a = z(7, 7); a[1:6, 1:6] = 1; a[3, 3] = 0; a[2, 2] = 0; cases["holes_touching_diagonally"] = a
    a = z(10, 10); a[2:8, 2:8] = 1; a[4:6, 4:6] = 0; a[4, 6] = 0; cases["hole_with_spur"] = a
    a = z(5, 7); a[1:4, 1:6] = 1; a[2, 2] = a[2, 4] = 0; cases["two_one_pixel_holes"] = a
    return cases


def _box_blur(x, r):
    """mean over a (2r+1)^2 window along the last two axes, edges replicated"""
    for ax in (-2, -1):
        p = np.pad(x, [(0, 0)] * (x.ndim - 2) + ([(r, r), (0, 0)] if ax == -2 else [(0, 0), (r, r)]), mode="edge")
        c = np.cumsum(p, axis=ax, dtype=np.float64)
        c = np.concatenate([np.zeros_like(np.take(c, [0], axis=ax)), c], axis=ax)
        n = x.shape[ax]
        x = (np.take(c, np.arange(2 * r + 1, n + 2 * r + 1), axis=ax) - np.take(c, np.arange(n), axis=ax)) / (2 * r + 1)
    return x


def prob_maps(seed, N, H, W, noise=2.0):
    """fp32 [N,1,H,W] probability maps whose 0.3-bitmap has text-box blobs, specks, broken edges and a few holes"""
    gt = db_batch(seed, N, H, W)["gt"]
    rng = np.random.RandomState(seed + 1)
    logit = (_box_blur(gt, 2) - 0.5) * 12.0 + noise * rng.standard_normal(gt.shape)
    return (1.0 / (1.0 + np.exp(-logit))).astype(np.float32)


def cv2_contours(bitmap):
    import cv2
    cs, _ = cv2.findContours((np.asarray(bitmap) != 0).astype(np.uint8) * 255, cv2.RETR_LIST, cv2.CHAIN_APPROX_NONE)
    return list(cs)


def digest(contours):
    """one hash of a contour list: number, order and points"""
    h = hashlib.sha256()
    for c in contours:
        c = np.ascontiguousarray(np.asarray(c).reshape(-1, 2), dtype=np.int32)
        h.update(np.int64(len(c)).tobytes())
        h.update(c.tobytes())
    return h.hexdigest()


# (name, seed, N, H, W, thresh, max_candidates, noise): the yaml's validation shape, odd sizes, a limit below and above the
# number of contours (the truncation keeps cv2's first ones), and low-noise maps whose contours are mostly text boxes (many
# candidates reach the score)
GPU_CASES = [
    ("val_4x576x1024_c1000", 11, 4, 576, 1024, 0.3, 1000, 2.0),
    ("val_4x576x1024_c100", 11, 4, 576, 1024, 0.3, 100, 2.0),
    ("odd_1x577x1023", 12, 1, 577, 1023, 0.3, 100000, 2.0),
    ("odd_3x33x47", 13, 3, 33, 47, 0.3, 1000, 2.0),
    ("square_16x640x640", 14, 16, 640, 640, 0.5, 1000, 2.0),
    ("clean_4x576x1024", 15, 4, 576, 1024, 0.3, 1000, 0.7),
]


def case_maps(name):
    for c in GPU_CASES:
        if c[0] == name:
            _, seed, N, H, W, thresh, maxc, noise = c
            return prob_maps(seed, N, H, W, noise), thresh, maxc
    raise KeyError(name)


def get_mini_boxes(contour):
    """The reference's get_mini_boxes (seg_detector_representer.py:125-145): the corners of cv2.minAreaRect as cv2.boxPoints gives
    them, stably sorted by x; of the two left corners the one with the smaller y comes first, of the two right ones the one with
    the smaller y second.  Returns ([4, 2] float32 corners, min(width, height))."""
    import cv2
    rect = cv2.minAreaRect(contour)
    by_x = sorted(cv2.boxPoints(rect), key=lambda corner: corner[0])
    left = (by_x[0], by_x[1]) if by_x[1][1] > by_x[0][1] else (by_x[1], by_x[0])     # (upper, lower)
    right = (by_x[2], by_x[3]) if by_x[3][1] > by_x[2][1] else (by_x[3], by_x[2])
    return np.array([left[0], right[0], right[1], left[1]]), min(rect[1])


def box_score_fast(score_map, corners):
    """The reference's box_score_fast (seg_detector_representer.py:156-168, int for the removed np.int): the mean of score_map
    under cv2.fillPoly of the corners on a mask over their bounding rows and columns (clipped to the map), corners shifted to
    the mask's origin and truncated with astype(np.int32)."""
    import cv2
    H, W = score_map.shape[:2]
    xs, ys = corners[:, 0], corners[:, 1]
    x0, x1 = (np.clip(f(xs).astype(int), 0, W - 1) for f in (lambda v: np.floor(v.min()), lambda v: np.ceil(v.max())))
    y0, y1 = (np.clip(f(ys).astype(int), 0, H - 1) for f in (lambda v: np.floor(v.min()), lambda v: np.ceil(v.max())))
    shifted = corners.copy()                         # float32: the shifts are exact, then truncated toward zero
    shifted[:, 0] = xs - x0
    shifted[:, 1] = ys - y0
    mask = np.zeros((y1 - y0 + 1, x1 - x0 + 1), np.uint8)
    cv2.fillPoly(mask, shifted.reshape(1, -1, 2).astype(np.int32), 1)
    return cv2.mean(score_map[y0:y1 + 1, x0:x1 + 1], mask)[0]


def reference_candidates(maps, thresh, maxc):
    """over cv2's kept contours (zero past the count): [N, maxc, 4, 2] corners and [N, maxc] ssides of get_mini_boxes, and
    [N, maxc] box_score_fast on the map where sside >= 3 (0 elsewhere) -- seg_detector_representer.py:80-94"""
    boxes = np.zeros((len(maps), maxc, 4, 2), np.float32)
    ssides = np.zeros((len(maps), maxc), np.float32)
    scores = np.zeros((len(maps), maxc), np.float64)
    for n, m in enumerate(maps):
        m = m.reshape(m.shape[-2:])
        for c, contour in enumerate(cv2_contours(m > np.float32(thresh))[:maxc]):
            boxes[n, c], ssides[n, c] = get_mini_boxes(contour)
            if ssides[n, c] >= 3:
                scores[n, c] = box_score_fast(m, boxes[n, c].reshape(-1, 2))
    return boxes, ssides, scores


# cases whose reference candidates are stored in the golden (the others are compared with cv2 where it is importable)
BOX_GOLDEN_CASES = ("val_4x576x1024_c1000", "odd_3x33x47", "clean_4x576x1024")


def reference(maps, thresh, maxc):
    """per image: (total contours, kept contours' digest) of cv2.findContours(maps > float32(thresh))[:maxc]"""
    out = []
    for m in maps:
        cs = cv2_contours(m.reshape(m.shape[-2:]) > np.float32(thresh))
        out.append((len(cs), digest(cs[:maxc])))
    return out
