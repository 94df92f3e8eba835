"""Generate tests/golden/db_targets_ref.npz with the REFERENCE's own MakeSegDetectionData and MakeBorderMap classes
(data/processes/make_seg_detection_data.py, make_border_map.py, loaded unmodified through oracle/ref_loader), their
shapely.geometry.Polygon and pyclipper.PyclipperOffset bound to the restatements of oracle/db_targets_port.py.  The per-polygon
status (not a reference output) comes from the oracle.

    python -m oracle.make_db_targets_golden

Cases are seeded (tests/db_targets_cases.py); images whose pad would be empty (the reference raises IndexError) are drawn
again.  gt, mask and thresh_mask are stored bit-packed; thresh_map as the bit-packed set of pixels that differ from
thresh_min and their float32 values in raster order, delta-coded by byte plane (encode_values); all compressed, so the file
stays well under 1 MB."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import db_targets_port as port  # noqa: E402
from tests.db_targets_cases import image_polygons  # noqa: E402

CASES = [  # name, seed, N, H, W, min / max polygons, dtype, share of odd quads
    ("b640", 1, 1, 640, 640, 6, 12, np.float64, 0.3),
    ("f32", 2, 2, 320, 480, 5, 12, np.float32, 0.5),
    ("wide", 3, 1, 576, 1024, 4, 8, np.float64, 0.3),
    ("odd", 4, 3, 256, 256, 5, 12, np.float64, 1.0),
]


def encode_values(v):
    """float32 values -> uint8 [4, n]: the byte planes of the successive differences (mod 2^32) of their bit patterns, which
    compress to about a quarter of the raw floats; tests/test_db_targets_gpu.py decodes them"""
    bits = v.astype(np.float32).view(np.uint32)
    d = np.diff(bits, prepend=np.uint32(0)).astype(np.uint32)
    return np.ascontiguousarray(d.view(np.uint8).reshape(-1, 4).T)


def reference_classes():
    from oracle import ref_loader
    if not ref_loader.install():
        raise SystemExit("reference tree not present")
    sys.modules["shapely.geometry"].Polygon = port.Polygon
    pc = sys.modules["pyclipper"]
    pc.PyclipperOffset, pc.JT_ROUND, pc.ET_CLOSEDPOLYGON = port.PyclipperOffset, port.JT_ROUND, port.ET_CLOSEDPOLYGON
    return (ref_loader.load("data.processes.make_seg_detection_data").MakeSegDetectionData(),
            ref_loader.load("data.processes.make_border_map").MakeBorderMap())


def main():
    seg, border = reference_classes()
    out = {}
    for name, seed, N, H, W, lo, hi, dtype, odd in CASES:
        rng = np.random.default_rng(seed)
        images = []
        while len(images) < N:
            polys, tags = image_polygons(rng, H, W, int(rng.integers(lo, hi + 1)), dtype, odd)
            want = port.make_targets(polys.copy(), tags, (H, W))
            if (want["status"] & port.PAD_EMPTY).any():
                continue
            data = dict(image=np.zeros((H, W, 3), np.float32), polygons=polys.copy(), ignore_tags=[bool(t) for t in tags],
                        filename="golden")
            with np.errstate(all="ignore"):
                data = border.process(seg.process(data))
            images.append((polys, tags, data, want["status"]))
        counts = np.array([len(p) for p, _, _, _ in images])
        out[name + "/size"] = np.array([N, H, W])
        out[name + "/counts"] = counts
        out[name + "/polygons_in"] = np.concatenate([p for p, _, _, _ in images]).reshape(-1, 4, 2)
        out[name + "/tags_in"] = np.concatenate([t for _, t, _, _ in images]).astype(bool).reshape(-1)
        out[name + "/polygons"] = np.concatenate([np.asarray(d["polygons"]) for _, _, d, _ in images]).reshape(-1, 4, 2)
        out[name + "/ignore_tags"] = np.concatenate([np.asarray(d["ignore_tags"], bool) for _, _, d, _ in images]).reshape(-1)
        out[name + "/status"] = np.concatenate([s for _, _, _, s in images]).astype(np.int32).reshape(-1)
        for k in ("gt", "mask", "thresh_mask"):
            out[name + "/" + k] = np.packbits(np.stack([np.asarray(d[k]).reshape(H, W) for _, _, d, _ in images]) != 0)
        tm = np.stack([d["thresh_map"] for _, _, d, _ in images]).astype(np.float32)
        off = tm != np.float32(0.3)                      # thresh_min outside every padded box
        out[name + "/thresh_map_at"] = np.packbits(off)
        out[name + "/thresh_map_planes"] = encode_values(tm[off])
    path = os.path.join(ROOT, "tests", "golden", "db_targets_ref.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
