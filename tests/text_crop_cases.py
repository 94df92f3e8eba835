"""Seeded inputs of the text-crop tests: textured images (uint8 and float32 HWC) and quads of every kind ImageCropper meets --
rotated boxes, axis-aligned and 45 degree ones, thin and tall ones, integer corners as boxes_from_maps returns them, and
degenerate ones (repeated corners, collinear corners, a point, sides under one pixel).  Also the host harness
(tests/host_harness/text_crop_core_host.cpp, the product's text_crop_core.cuh compiled with g++)."""
import ctypes
import os
import shutil
import subprocess

import numpy as np

KINDS = ("rotated", "axis", "diag45", "thin", "tall", "int", "repeat", "collinear", "point", "subpixel")


def image(rng, h, w, dtype=np.uint8):
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    base = np.stack([127 + 100 * np.sin(x / 5.0 + c) * np.cos(y / 9.0 - c) for c in range(3)], -1)
    base += 40 * ((x // 8 + y // 8) % 2)[..., None] + rng.normal(0, 12, (h, w, 3))
    img = np.clip(base, 0, 255)
    if dtype == np.uint8:
        return img.astype(np.uint8)
    return (img + rng.random((h, w, 3))).astype(np.float32)


def quad(rng, kind, h, w):
    """One [4, 2] float32 quad of the given kind inside (or slightly past) an h x w image"""
    cx, cy = rng.uniform(-0.05 * w, 1.05 * w), rng.uniform(-0.05 * h, 1.05 * h)
    if kind in ("rotated", "thin", "tall", "int", "axis", "diag45"):
        bw, bh = rng.uniform(4, 0.6 * w), rng.uniform(3, 0.3 * h)
        if kind == "thin":
            bh = rng.uniform(0.6, 3)
        if kind == "tall":
            bw, bh = rng.uniform(3, 0.15 * w), rng.uniform(10, 0.8 * h)
        a = {"axis": 0.0, "diag45": np.pi / 4 * rng.choice([1, -1, 3])}.get(kind, rng.uniform(-np.pi, np.pi))
        c, s = np.cos(a), np.sin(a)
        pts = np.array([(-bw / 2, -bh / 2), (bw / 2, -bh / 2), (bw / 2, bh / 2), (-bw / 2, bh / 2)]) @ [[c, s], [-s, c]] + (cx, cy)
        pts += rng.normal(0, 0.8, pts.shape) * (kind == "rotated")
        if kind in ("int", "axis"):
            pts = np.round(pts)
        return pts.astype(np.float32)
    if kind == "repeat":
        p = rng.uniform(0, 1, (3, 2)) * (w, h)
        return p[[0, 1, 1, 2]].astype(np.float32)
    if kind == "collinear":
        d = rng.normal(0, 1, 2)
        t = np.sort(rng.uniform(-0.3, 0.3, 4)) * max(h, w)
        pts = np.array([(cx, cy) + ti * d for ti in t])
        if rng.random() < 0.5:
            pts = np.round(pts)
        return pts.astype(np.float32)
    if kind == "point":
        return np.tile(np.round([cx, cy]), (4, 1)).astype(np.float32)
    if kind == "subpixel":
        bw, bh = rng.uniform(0.1, 0.99), rng.uniform(2, 40)
        if rng.random() < 0.5:
            bw, bh = bh, bw
        return np.array([(cx, cy), (cx + bw, cy), (cx + bw, cy + bh), (cx, cy + bh)], np.float32)
    raise ValueError(kind)


def quads(seed, count, h=720, w=1280):
    """count seeded quads cycling through KINDS -> ([count, 4, 2] float32, kinds)"""
    rng = np.random.default_rng(seed)
    kinds = [KINDS[i % len(KINDS)] for i in range(count)]
    return np.array([quad(rng, k, h, w) for k in kinds], np.float32).reshape(count, 4, 2), kinds


# ---- the host harness ----

def build_harness(out_dir):
    here = os.path.dirname(os.path.abspath(__file__))
    gxx = shutil.which("g++")
    if not gxx:
        return None
    so = os.path.join(str(out_dir), "libtext_crop_core_host.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                           "-I", os.path.join(here, "..", "megreader_b200", "csrc"),
                           os.path.join(here, "host_harness", "text_crop_core_host.cpp"), "-o", so])
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def host_setup(lib, q, img_h, img_w, mode="resize", image_size=(64, 512)):
    """-> dict(box [k, 4, 2], sides [k, 2] float32, size [k, 4] (crop w, h, resize input h, w), turned, valid_w, flags, P, M)"""
    q = np.ascontiguousarray(q, np.float32).reshape(-1, 4, 2)
    k = len(q)
    box, sides = np.zeros((k, 4, 2), np.float32), np.zeros((k, 2), np.float32)
    size, ints = np.zeros((k, 4), np.int32), np.zeros((k, 3), np.int32)
    P, M = np.zeros((k, 3, 3)), np.zeros((k, 3, 3))
    lib.host_setup(_p(q), k, int(img_h), int(img_w), int(mode == "pad"), int(image_size[0]), int(image_size[1]), _p(box), _p(sides),
                   _p(size), _p(ints), _p(P), _p(M))
    return dict(box=box, sides=sides, size=size, turned=ints[:, 0].astype(bool), valid_w=ints[:, 1], flags=ints[:, 2], P=P, M=M)


def host_warp(lib, img, P, dsize):
    img = np.ascontiguousarray(img)
    P = np.ascontiguousarray(P, np.float64)
    out = np.zeros((dsize[1], dsize[0], 3), np.float32)
    lib.host_warp(_p(img), int(img.dtype == np.float32), img.shape[0], img.shape[1], _p(P), int(dsize[0]), int(dsize[1]), _p(out))
    return out


def host_crop(lib, img, q, image_size=(64, 512), mode="resize"):
    img = np.ascontiguousarray(img)
    q = np.ascontiguousarray(q, np.float32)
    out = np.zeros((image_size[0], image_size[1], 3), np.float32)
    lib.host_crop(_p(img), int(img.dtype == np.float32), img.shape[0], img.shape[1], _p(q), int(mode == "pad"), int(image_size[0]),
                  int(image_size[1]), _p(out))
    return out
