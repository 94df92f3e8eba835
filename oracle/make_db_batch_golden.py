"""Generate tests/golden/db_batch_ref.npz with the REFERENCE's own RandomCropData, MakeICDARData and NormalizeImage
(data/processes/random_crop_data.py, make_icdar_data.py, normalize_image.py, loaded unmodified through oracle/ref_loader)
after the augmentation of oracle/db_batch_port.py.  np.random.choice in random_crop_data's namespace is patched to take its
picks from the draws (axis[min(floor(u * len), len - 1)]), and crop_area is wrapped to record the rectangle it returns.

    python -m oracle.make_db_batch_golden

Per case (tests/db_batch_cases.py) the file stores the draws, the crop rectangle, scale and which crop_area call found it,
the kept quads and tags, and for the normalised image a seeded sample of pixels (tests.db_batch_cases.pixel_sample) and the
per-channel sums: both as the host harness computes them (the device's target, bit for bit) and as the reference's cv2
chain computes them."""
import os
import sys
import tempfile
from collections import OrderedDict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import db_batch_port as port  # noqa: E402
from tests import db_batch_cases as C  # noqa: E402


def reference_processes():
    from oracle import make_db_targets_golden, ref_loader
    # data.processes imports every process module: bind shapely / pyclipper to their restatements first, as the targets'
    # golden does, so that whichever loads the package first leaves it usable for the other
    make_db_targets_golden.reference_classes()
    rc = ref_loader.load("data.processes.random_crop_data")
    icdar = ref_loader.load("data.processes.make_icdar_data")
    norm = ref_loader.load("data.processes.normalize_image")
    return rc, icdar.MakeICDARData(), norm.NormalizeImage()


def reference_train(rc, icdar, norm, image, polys, tags, u):
    """AugmentDetectionData's output (restated) through the reference's own RandomCropData / MakeICDARData / NormalizeImage"""
    img, p, _ = port.augment(image.astype(np.float32), polys, u)
    picks = port.Picks(u, 10)

    class _Random:
        @staticmethod
        def choice(axis, size=2):
            return picks(axis, size)
    crop = RandomCropDataRecorder(rc, picks)
    saved = rc.np
    rc.np = type("np_with_draws", (), {k: getattr(np, k) for k in ("zeros", "int32", "round", "where", "min", "max", "clip", "array")})
    rc.np.random = _Random
    try:
        data = crop.process(OrderedDict(image=img, polys=[dict(points=q.tolist(), ignore=bool(t), text="###" if t else "x")
                                                          for q, t in zip(p, tags)], shape=image.shape[:2], filename="", data_id=""))
    finally:
        rc.np = saved
    data = icdar.process(data)
    data = norm.process(data)
    return data, crop.rect, crop.round


class RandomCropDataRecorder:
    """The reference's RandomCropData(size=[640, 640], max_tries=10) with crop_area wrapped to record its result"""

    def __init__(self, rc, picks):
        self.inner = rc.RandomCropData(size=[640, 640], max_tries=10)
        self.rect, self.round, self.calls = None, None, 0
        inner_area = self.inner.crop_area

        def area(img, polys, width=None, height=None):
            self.calls += 1
            picks.calls = 0 if width is not None else 20
            r = inner_area(img, polys, width, height)
            if self.rect is None or width is not None:
                self.rect = tuple(int(v) for v in r)
            return r
        self.inner.crop_area = area

    def process(self, data):
        return self.inner.process(data)


def main():
    rc, icdar, norm = reference_processes()
    lib = C.build_harness(tempfile.mkdtemp())
    out = {}
    for i, (name, *_) in enumerate(C.CASES):
        c = C.case(name)
        h, w = c["image"].shape[:2]
        g = C.host_geometry(lib, c["mode"], h, w, c["polys"], c["tags"], c["draws"])
        host_img = C.host_output(lib, c["mode"], c["image"], g, c["draws"])
        if c["mode"] == "train":
            data, rect, _ = reference_train(rc, icdar, norm, c["image"], c["polys"], c["tags"], c["draws"])
            o = port.train_sample(c["image"], c["polys"], c["tags"], c["draws"])
            ref_img = data["image"].numpy() if hasattr(data["image"], "numpy") else np.asarray(data["image"])
            polys = np.asarray(data["polygons"], np.float64).reshape(-1, 4, 2)
            tags = np.asarray(data["ignore_tags"], np.uint8)
            scale = float(o["scale"])
            assert rect == tuple(o["crop"]), (name, rect, o["crop"])
            out[name + "/round"] = np.int32(o["round"])
            out[name + "/crop"] = np.array(rect, np.int32)
        else:
            o = port.validate_sample(c["image"], c["polys"], c["tags"])
            ref_img, polys, tags, scale = o["image"], o["polygons"], o["ignore_tags"], 1.0
            out[name + "/crop"] = np.array([0, 0, 1024, 576], np.int32)
        ref_img = np.asarray(ref_img, np.float32)
        idx = C.pixel_sample(i, ref_img.shape)
        out[name + "/draws"] = c["draws"]
        out[name + "/scale"] = np.float64(scale)
        out[name + "/polygons"] = polys
        out[name + "/ignore_tags"] = tags
        out[name + "/host_pixels"] = host_img.reshape(-1)[idx]
        out[name + "/host_sums"] = host_img.astype(np.float64).sum((1, 2))
        out[name + "/ref_pixels"] = ref_img.reshape(-1)[idx]
        out[name + "/ref_sums"] = ref_img.astype(np.float64).sum((1, 2))
        print(name, out[name + "/crop"], scale, len(polys), float(np.abs(host_img - ref_img).max()))
    path = os.path.join(ROOT, "tests", "golden", "db_batch_ref.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
