"""TEST INFRASTRUCTURE ONLY (never imported by the product): CPU restatement of seg_detector_db.yaml's data processes
before the targets, from the same draws as megreader_b200.db_batch.

    augment(image, polys, u, ...)        AugmentDetectionData: imgaug's Fliplr / Affine(rotate) / Resize restated in numpy after
                                         imgaug 0.4.0, with cv2 doing the flip, cv2.warpAffine and cv2.resize (INTER_CUBIC)
    crop_area(...) / random_crop(...)    RandomCropData (data/processes/random_crop_data.py) restated, np.random.choice's picks
                                         taken from the draws
    train_sample / validate_sample       the whole chain, then MakeICDARData and NormalizeImage

The rotation's sin and cos come from the same Taylor series as csrc/db_batch_core.cuh, so the matrices agree bit for bit."""
import math

import cv2
import numpy as np

RGB_MEAN = np.array([122.67891434, 116.66876762, 104.00698793])


def sin_cos(r):
    r2 = r * r
    ps = pc = 1.0
    for k in range(16, 0, -1):
        ps = 1.0 - (r2 * ps) * (1.0 / ((2.0 * k) * (2.0 * k + 1.0)))
        pc = 1.0 - (r2 * pc) * (1.0 / ((2.0 * k - 1.0) * (2.0 * k)))
    return r * ps, pc


def rotation_matrix(deg, w, h):
    """imgaug's Affine(rotate=deg): about (w / 2 - 0.5, h / 2 - 0.5), skimage's rotation sense; forward [2, 3] float64"""
    s, c = sin_cos(deg * (math.pi / 180.0))
    cx, cy = w / 2.0 - 0.5, h / 2.0 - 0.5
    return np.array([[c, -s, (cx - c * cx) + s * cy], [s, c, (cy - s * cx) - c * cy]])


def params(u, rotate=(-10, 10), scale=(0.5, 3.0), flip_p=0.5):
    u = np.asarray(u, np.float32)
    flip = float(u[0]) < flip_p
    deg = rotate[0] + float(u[1]) * (rotate[1] - rotate[0])
    s = scale[0] + float(u[2]) * (scale[1] - scale[0])
    return flip, deg, s


def augment(image, polys, u, rotate=(-10, 10), scale=(0.5, 3.0), flip_p=0.5):
    """float32 HWC image, float64 [k, 4, 2] quads -> (augmented image, quads, (flip, deg, hs, ws))"""
    h, w = image.shape[:2]
    flip, deg, s = params(u, rotate, scale, flip_p)
    img = cv2.flip(image, 1) if flip else image
    M = rotation_matrix(deg, w, h)
    img = cv2.warpAffine(img, M, (w, h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    hs, ws = max(1, int(round(s * h))), max(1, int(round(s * w)))
    img = cv2.resize(img, (ws, hs), interpolation=cv2.INTER_CUBIC)
    p = np.array(polys, np.float64).reshape(-1, 2).copy()
    if flip:
        p[:, 0] = w - p[:, 0]
    x = (M[0, 0] * p[:, 0] + M[0, 1] * p[:, 1]) + M[0, 2]
    y = (M[1, 0] * p[:, 0] + M[1, 1] * p[:, 1]) + M[1, 2]
    p = np.stack([(x / w) * ws, (y / h) * hs], 1).reshape(-1, 4, 2)
    return img, p, (flip, deg, hs, ws)


def resize_points(polys, h, w, hs, ws):
    p = np.array(polys, np.float64).reshape(-1, 2)
    return np.stack([(p[:, 0] / w) * ws, (p[:, 1] / h) * hs], 1).reshape(-1, 4, 2)


class Picks:
    """np.random.choice(axis, size=2) from the draws: axis[min(floor(u * len), len - 1)], in draw order per try"""

    def __init__(self, u, max_tries):
        self.u, self.max_tries, self.calls = np.asarray(u, np.float32), max_tries, 0

    def __call__(self, axis, size=2):
        rnd, t, xy = divmod(self.calls, 2 * self.max_tries)[0], (self.calls // 2) % self.max_tries, self.calls % 2
        self.calls += 1
        base = 3 + 4 * (rnd * self.max_tries + t) + 2 * xy
        n = len(axis)
        return np.array([axis[min(max(int(math.floor(float(self.u[base + j]) * n)), 0), n - 1)] for j in range(size)])


def outside(poly, x, y, w, h):
    p = np.asarray(poly)
    return p[:, 0].max() < x or p[:, 0].min() > x + w or p[:, 1].max() < y or p[:, 1].min() > y + h


def crop_area(h, w, care, picks, size, max_tries, min_ratio):
    """RandomCropData.crop_area; returns (x, y, w, h, round) with round 0 / 1 for the call that found it, 2 for the whole
    image"""
    def one_call(fixed):
        cols, rows = np.zeros(w, bool), np.zeros(h, bool)
        for q in care:
            r = np.round(q, 0).astype(np.int32)
            cols[r[:, 0].min():r[:, 0].max()] = True
            rows[r[:, 1].min():r[:, 1].max()] = True
        xs, ys = np.flatnonzero(~cols), np.flatnonzero(~rows)
        if len(xs) == 0 or len(ys) == 0:
            return None
        for _ in range(max_tries):
            xx = picks(xs)
            x0 = xx.min()
            x1 = x0 + size if fixed else xx.max()
            x0, x1 = np.clip(x0, 0, w - 1), np.clip(x1, 0, w - 1)
            yy = picks(ys)
            y0 = yy.min()
            y1 = y0 + size if fixed else yy.max()
            y0, y1 = np.clip(y0, 0, h - 1), np.clip(y1, 0, h - 1)
            if x1 - x0 < min_ratio * w or y1 - y0 < min_ratio * h:
                continue
            if any(not outside(q, x0, y0, x1 - x0, y1 - y0) for q in care):
                return int(x0), int(y0), int(x1 - x0), int(y1 - y0)
        return None
    for rnd, fixed in ((0, True), (1, False)):
        picks.calls = 2 * max_tries * rnd
        r = one_call(fixed)
        if r is not None:
            return r + (rnd,)
    return (0, 0, w, h, 2)


def random_crop(img, polys, tags, u, size=(640, 640), max_tries=10, min_ratio=0.1):
    """RandomCropData: -> (canvas float32 [size[1], size[0], 3], kept quads float64, kept tags, (x, y, w, h), scale, round)"""
    hs, ws = img.shape[:2]
    care = [q for q, t in zip(polys, tags) if not t]
    cx, cy, cw, ch, rnd = crop_area(hs, ws, care, Picks(u, max_tries), size[0], max_tries, min_ratio)
    scale = min(size[0] / cw, size[1] / ch)
    oh, ow = int(ch * scale), int(cw * scale)
    canvas = np.zeros((size[1], size[0], 3), img.dtype)
    canvas[:oh, :ow] = cv2.resize(img[cy:cy + ch, cx:cx + cw], (ow, oh))
    kept, ktags = [], []
    for q, t in zip(polys, tags):
        p = (np.asarray(q, np.float64) - (cx, cy)) * scale
        if not outside(p, 0, 0, ow, oh):
            kept.append(p)
            ktags.append(t)
    return canvas, np.array(kept, np.float64).reshape(-1, 4, 2), np.array(ktags, np.uint8), (cx, cy, cw, ch), scale, rnd


def normalize(img):
    return ((img.astype(np.float32) - RGB_MEAN).astype(np.float32) / np.float32(255.)).transpose(2, 0, 1).astype(np.float32)


def train_sample(image, polys, tags, u, size=(640, 640), max_tries=10, min_ratio=0.1, rotate=(-10, 10), scale=(0.5, 3.0),
                 flip_p=0.5):
    img, p, (flip, deg, hs, ws) = augment(image.astype(np.float32), polys, u, rotate, scale, flip_p)
    canvas, kept, ktags, crop, sc, rnd = random_crop(img, p, np.asarray(tags, np.uint8), u, size, max_tries, min_ratio)
    return dict(image=normalize(canvas), polygons=kept, ignore_tags=ktags, crop=crop, scale=sc, round=rnd, flip=flip, deg=deg,
                hs=hs, ws=ws, augmented=p, shape=image.shape[:2])


def validate_sample(image, polys, tags, size=(576, 1024)):
    h, w = image.shape[:2]
    img = cv2.resize(image.astype(np.float32), (size[1], size[0]), interpolation=cv2.INTER_CUBIC)
    return dict(image=normalize(img), polygons=resize_points(polys, h, w, size[0], size[1]),
                ignore_tags=np.asarray(tags, np.uint8), shape=(h, w))
