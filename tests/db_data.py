"""Seeded synthetic DB (Differentiable Binarization) batches, numpy only: the targets data/processes/make_seg_detection_data.py and
make_border_map.py would produce for random text boxes, without cv2 or polygon clipping.

    gt          [N,1,H,W]  1 inside the (shrunk) text boxes, 5-15 % of the pixels of each image
    mask        [N,H,W]    1 except a few ignore boxes
    thresh_map  [N,H,W]    0.3 .. 0.7 on a border band around each box (0.7 on the box edge), 0.3 elsewhere
    thresh_mask [N,H,W]    1 on the border bands
Boxes are axis-aligned or rotated rectangles.  Used by the benchmark (bench_trunks.py config 6) and the GPU tests."""
import numpy as np


def _box(rng, H, W, scale):
    cy, cx = rng.uniform(0, H), rng.uniform(0, W)
    h = rng.uniform(0.03, 0.12) * scale
    w = h * rng.uniform(1.5, 8.0)
    ang = 0.0 if rng.rand() < 0.5 else rng.uniform(-np.pi / 4, np.pi / 4)
    return cy, cx, h, w, ang


def _box_coords(yy, xx, box):
    cy, cx, h, w, ang = box
    c, s = np.cos(ang), np.sin(ang)
    dy, dx = yy - cy, xx - cx
    u = dx * c + dy * s           # along the box
    v = -dx * s + dy * c          # across
    return np.abs(u) - w / 2, np.abs(v) - h / 2


def db_batch(seed, N, H, W, pos_frac=(0.05, 0.15)):
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32) + 0.5
    scale = float(min(H, W))
    gt = np.zeros((N, 1, H, W), np.float32)
    mask = np.ones((N, H, W), np.float32)
    tmap = np.full((N, H, W), 0.3, np.float32)
    tmask = np.zeros((N, H, W), np.float32)
    for n in range(N):
        target = rng.uniform(*pos_frac)
        for _ in range(400):
            if gt[n, 0].mean() >= target:
                break
            box = _box(rng, H, W, scale)
            du, dv = _box_coords(yy, xx, box)
            inside = (du <= 0) & (dv <= 0)
            band_w = max(1.0, 0.4 * box[2])
            out_d = np.sqrt(np.maximum(du, 0) ** 2 + np.maximum(dv, 0) ** 2)          # distance outside the box
            in_d = np.where(inside, -np.maximum(du, dv), 0.0)                           # distance inside the box
            d = np.where(inside, in_d, out_d)
            band = d <= band_w
            val = 0.7 - 0.4 * np.clip(d / band_w, 0.0, 1.0)
            tmap[n] = np.where(band, np.maximum(tmap[n], val), tmap[n])
            tmask[n][band] = 1.0
            shrunk = inside & (in_d >= 0.2 * band_w)
            gt[n, 0][shrunk] = 1.0
        for _ in range(rng.randint(1, 4)):                                              # ignore regions
            du, dv = _box_coords(yy, xx, _box(rng, H, W, scale * 0.5))
            mask[n][(du <= 0) & (dv <= 0)] = 0.0
    return {"gt": gt, "mask": mask, "thresh_map": tmap, "thresh_mask": tmask}


def db_images(seed, N, H, W):
    """Images at the scale of the yaml's NormalizeImage output (what the trunk sees): seeded normal noise."""
    rng = np.random.RandomState(seed)
    return (rng.standard_normal((N, 3, H, W)) * 0.5).astype(np.float32)
