"""Seeded polygon sets for the DB target tests: per image a [n, 4, 2] array and its ignore tags, covering the cases real
crops produce (rotated text boxes 10 to 80 px high, quads clipped at the crop border with zero-length edges) and the edge
cases of MakeSegDetectionData / MakeBorderMap (sub-8 px text, |area| < 1, duplicate corners, concave and bow-tie quads,
overlaps, polygons wholly outside the image)."""
import numpy as np


def rotated_box(rng, H, W, lo=10, hi=80):
    h = rng.uniform(lo, hi)
    w = rng.uniform(h, min(6 * h, 0.9 * W))
    cx, cy = rng.uniform(-0.05 * W, 1.05 * W), rng.uniform(-0.05 * H, 1.05 * H)
    a = rng.uniform(-np.pi / 4, np.pi / 4)
    c, s = np.cos(a), np.sin(a)
    pts = np.array([[-w / 2, -h / 2], [w / 2, -h / 2], [w / 2, h / 2], [-w / 2, h / 2]])
    out = pts @ np.array([[c, s], [-s, c]]) + [cx, cy]
    return out[::-1] if rng.random() < 0.3 else out


def odd_quad(rng, H, W):
    kind = rng.integers(0, 8)
    b = rotated_box(rng, H, W)
    if kind == 0:                                  # sub-8 px text
        b = rotated_box(rng, H, W, 2, 7.9)
    elif kind == 1:                                # |area| < 1
        x, y = rng.uniform(0, W), rng.uniform(0, H)
        b = np.array([[x, y], [x + rng.uniform(0, 30), y], [x + rng.uniform(0, 30), y + rng.uniform(0, 0.03)], [x, y]])
    elif kind == 2:                                # duplicate corners (a triangle)
        b[2] = b[1]
    elif kind == 3:                                # concave: one corner pulled inwards
        c = b.mean(0)
        b[1] = c + (b[1] - c) * rng.uniform(-0.3, 0.4)
    elif kind == 4:                                # bow-tie
        b[[1, 2]] = b[[2, 1]]
    elif kind == 5:                                # crossing the border on purpose
        b += [rng.choice([-1, 1]) * W * 0.5, 0]
    elif kind == 6:                                # thin sliver (shrink may be empty)
        p = rng.uniform([0, 0], [W, H])
        d = rng.uniform(20, 200)
        t = rng.uniform(0, np.pi)
        u = np.array([np.cos(t), np.sin(t)]) * d
        v = np.array([np.cos(t + 0.08), np.sin(t + 0.08)]) * rng.uniform(8, 12)
        b = np.array([p, p + u, p + u + v, p + v])
    else:                                          # integer corners on the border (zero-length edges after clipping)
        b = np.round(b)
        b[:, 0] = np.where(rng.random(4) < 0.5, -5, b[:, 0])
    return b


def image_polygons(rng, H, W, n, dtype=np.float64, odd=0.3):
    polys = [odd_quad(rng, H, W) if rng.random() < odd else rotated_box(rng, H, W) for _ in range(n)]
    polys = np.array(polys, dtype=dtype).reshape(n, 4, 2)
    tags = rng.random(n) < 0.05
    return polys, tags


def batch(seed, N, H, W, nmin, nmax, dtype=np.float64, odd=0.3):
    rng = np.random.default_rng(seed)
    return [image_polygons(rng, H, W, int(rng.integers(nmin, nmax + 1)), dtype, odd) for _ in range(N)]
