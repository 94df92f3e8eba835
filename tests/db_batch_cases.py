"""Seeded inputs of the DB input-batch tests: textured uint8 HWC images (gradients, stripes and noise, so every resampling
step changes the pixels) with text-like quads, and draws that force the cases RandomCropData distinguishes.  Everything
regenerates from the seed on any machine."""
import numpy as np

from tests.db_targets_cases import rotated_box

MAX_H, MAX_W = 480, 640          # the largest declared input of the golden cases

# name, seed, mode, h, w, quads, share ignored, overrides (draw index -> value; "round1": every first-round x pick; "edge":
# boxes at the top left border; "right": all boxes in the right quarter, beyond a 640 crop from the left edge)
CASES = [
    ("crop640", 1, "train", 480, 640, 12, 0.2, {2: 0.9}),
    ("no_care", 2, "train", 300, 400, 6, 1.0, {}),
    ("second_round", 7, "train", 360, 500, 3, 0.0, {"round1": 0.0, 2: 1.0, "right": True}),
    ("negative", 4, "train", 320, 420, 10, 0.1, {1: 0.0, 0: 0.9, "edge": True}),
    ("scale3_max", 5, "train", MAX_H, MAX_W, 14, 0.2, {2: 1.0}),
    ("dropped", 6, "train", 400, 560, 14, 0.3, {2: 0.8}),
    ("flip_small", 7, "train", 200, 260, 5, 0.4, {0: 0.1, 2: 0.05}),
    ("validate", 8, "validate", 410, 530, 9, 0.3, {}),
]


def image(rng, h, w):
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    base = np.stack([127 + 100 * np.sin(x / 7.0 + c) * np.cos(y / 11.0 - c) for c in range(3)], -1)
    base += 40 * ((x // 16 + y // 16) % 2)[..., None] + rng.normal(0, 12, (h, w, 3))
    return np.clip(base, 0, 255).astype(np.uint8)


def quads(rng, h, w, n, edge=False, right=False):
    q = [rotated_box(rng, h, w, 8, max(9, min(60, h / 4))) for _ in range(n)]
    if right:
        q = [b - [b[:, 0].min() - rng.uniform(0.75, 0.85) * w, 0] for b in q]
    if edge:                       # boxes touching the left and top borders: the rotation moves their corners below zero
        for i in range(0, n, 2):
            q[i] = q[i] - q[i].min(0) + rng.uniform(0, 2, 2)
    return np.array(q, np.float64).reshape(n, 4, 2)


def draws(rng, mode, overrides, max_tries=10):
    u = rng.random(3 + 8 * max_tries).astype(np.float32)
    for k, v in overrides.items():
        if k == "round1":
            for t in range(max_tries):
                u[3 + 4 * t:3 + 4 * t + 2] = v
                u[3 + 4 * t + 2:3 + 4 * t + 4] = 0.5
        elif isinstance(k, int):
            u[k] = v
    return u if mode == "train" else np.zeros(0, np.float32)


def case(name):
    _, seed, mode, h, w, n, ign, ov = next(c for c in CASES if c[0] == name)
    rng = np.random.default_rng(seed)
    img = image(rng, h, w)
    q = quads(rng, h, w, n, bool(ov.get("edge")), bool(ov.get("right")))
    tags = (rng.random(n) < ign).astype(np.uint8)
    return dict(mode=mode, image=img, polys=q, tags=tags, draws=draws(rng, mode, ov))


def polygon_sets(seed, count):
    """Many seeded (h, w, quads, tags, draws) for the crop rule alone (no pixels)"""
    rng = np.random.default_rng(seed)
    for i in range(count):
        h, w = int(rng.integers(100, 900)), int(rng.integers(100, 900))
        n = int(rng.integers(0, 25))
        q = quads(rng, h, w, n, edge=i % 3 == 0) if n else np.zeros((0, 4, 2))
        tags = (rng.random(n) < rng.choice([0.0, 0.3, 1.0])).astype(np.uint8)
        u = rng.random(83).astype(np.float32)
        if i % 5 == 0:
            for t in range(10):
                u[3 + 4 * t:3 + 4 * t + 2] = 0.9999
        yield h, w, q, tags, u


# ---- the host harness (tests/host_harness/db_batch_core_host.cpp: the product's db_batch_core.cuh compiled with g++) ----

def build_harness(out_dir):
    import ctypes
    import os
    import shutil
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    gxx = shutil.which("g++")
    if not gxx:
        return None
    so = os.path.join(str(out_dir), "libdb_batch_core_host.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                           "-I", os.path.join(here, "..", "megreader_b200", "csrc"),
                           os.path.join(here, "host_harness", "db_batch_core_host.cpp"), "-o", so])
    return ctypes.CDLL(so)


def _p(a):
    import ctypes
    return a.ctypes.data_as(ctypes.c_void_p)


def host_geometry(lib, mode, h, w, polys, tags, u, size=(640, 640), val_size=(576, 1024), max_tries=10, min_ratio=0.1,
                  rotate=(-10, 10), scale=(0.5, 3.0), flip_p=0.5):
    """-> dict(hs, ws, flip, crop (x, y, w, h), oh, ow, scale, augmented [k, 4, 2], polygons (kept), ignore_tags (kept))"""
    import ctypes
    polys = np.ascontiguousarray(polys, np.float64).reshape(-1, 4, 2)
    tags = np.ascontiguousarray(tags, np.uint8)
    k = len(polys)
    u = np.ascontiguousarray(u if len(u) else np.zeros(3 + 8 * max_tries), np.float32)
    ints = np.zeros(9, np.int32)
    sc = ctypes.c_double(0)
    aug, out, keep = np.zeros((k, 4, 2)), np.zeros((k, 4, 2)), np.zeros(k, np.uint8)
    out_h, out_w = (size[1], size[0]) if mode == "train" else val_size
    d = ctypes.c_double
    lib.host_geometry(int(mode != "train"), out_h, out_w, max_tries, d(min_ratio), d(flip_p), d(rotate[0]), d(rotate[1]), d(scale[0]),
                      d(scale[1]), _p(u), h, w, _p(polys), _p(tags), k, _p(ints), ctypes.byref(sc), _p(aug), _p(out), _p(keep))
    keep = keep.astype(bool)
    return dict(hs=int(ints[0]), ws=int(ints[1]), flip=bool(ints[2]), crop=tuple(int(v) for v in ints[3:7]), oh=int(ints[7]),
                ow=int(ints[8]), scale=sc.value, augmented=aug, polygons=out[keep], ignore_tags=tags[keep], ints=ints)


def host_output(lib, mode, image, geom, u, size=(640, 640), val_size=(576, 1024), rotate=(-10, 10)):
    """The normalised [3, H, W] image as the device computes it, from a uint8 or float32 HWC image"""
    import ctypes
    img = np.ascontiguousarray(image, np.float32)
    h, w = img.shape[:2]
    out_h, out_w = (size[1], size[0]) if mode == "train" else val_size
    out = np.zeros((3, out_h, out_w), np.float32)
    u = np.ascontiguousarray(u if len(u) else np.zeros(3), np.float32)
    lib.host_output(int(mode != "train"), out_h, out_w, ctypes.c_double(rotate[0]), ctypes.c_double(rotate[1]), _p(u), _p(img), h, w,
                    _p(np.ascontiguousarray(geom["ints"])), ctypes.c_double(geom["scale"]), _p(out))
    return out


def pixel_sample(seed, shape, count=4096):
    """A fixed seeded sample of flat indices into a [3, H, W] image"""
    return np.random.default_rng(seed).integers(0, int(np.prod(shape)), count)
