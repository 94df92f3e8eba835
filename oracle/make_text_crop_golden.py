"""Generate tests/golden/text_crop_ref.npz with the REFERENCE's own ImageCropper (data/crop_file_dataset.py, loaded unmodified
through oracle/ref_loader).  Its module's cv2 is bound to a proxy whose warpPerspective takes (int(w), int(h)) for dsize: the
reference passes numpy float32 sides, which cv2 4.x refuses.  Nothing else changes.

    python -m oracle.make_text_crop_golden

Per case (uint8 and float32 images, both modes, tests/text_crop_cases.py's quads) the file stores the quad, a seeded sample of
the crop's values with cv2's optimisations off and with its defaults, and the crop's per-channel sums."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import text_crop_cases as C  # noqa: E402


class _Cv2IntDsize:
    """cv2 with warpPerspective's dsize truncated to int, as cv2 3.x accepted float sizes"""

    def __init__(self, cv2):
        self._cv2 = cv2

    def __getattr__(self, name):
        return getattr(self._cv2, name)

    def warpPerspective(self, image, mat, dsize, *args, **kwargs):
        return self._cv2.warpPerspective(image, mat, (int(dsize[0]), int(dsize[1])), *args, **kwargs)


def reference_cropper(image_size, mode):
    import cv2
    from oracle import ref_loader
    mod = ref_loader.load("data.crop_file_dataset")
    if not isinstance(mod.cv2, _Cv2IntDsize):
        mod.cv2 = _Cv2IntDsize(cv2)
    cropper = mod.ImageCropper(image_size=list(image_size), mode=mode)
    # crop() calls the ResizeImage process on an array; the process's own resize is what it means
    # ResizeImage(image_size, mode) binds image_size to its `cmd` argument and keeps its default size; use the cropper's
    cropper.resize.image_size = list(image_size)
    cropper.resize = cropper.resize.resize_or_pad
    return cropper


CASES = [("u8_resize", np.uint8, "resize", (32, 100)), ("f32_resize", np.float32, "resize", (64, 256)),
         ("u8_pad", np.uint8, "pad", (32, 100)), ("f32_pad", np.float32, "pad", (32, 100))]
SAMPLES = 256


def case_inputs(i, dtype):
    rng = np.random.default_rng(100 + i)
    img = C.image(rng, 140, 210, dtype)
    q, kinds = C.quads(200 + i, 40, 140, 210)
    return img, q, kinds


def main():
    import cv2
    out = {}
    for i, (name, dtype, mode, size) in enumerate(CASES):
        img, q, kinds = case_inputs(i, dtype)
        cropper = reference_cropper(size, mode)
        idx = np.random.default_rng(i).choice(size[0] * size[1] * 3, SAMPLES, replace=False)
        plain, dflt, sums = [], [], []
        for k in range(len(q)):
            cv2.setUseOptimized(False)
            a = np.asarray(cropper.crop(img, q[k]), np.float32)
            cv2.setUseOptimized(True)
            b = np.asarray(cropper.crop(img, q[k]), np.float32)
            plain.append(a.reshape(-1)[idx])
            dflt.append(b.reshape(-1)[idx])
            sums.append(a.astype(np.float64).sum((0, 1)))
        out[name + "/quads"] = q
        out[name + "/index"] = idx
        out[name + "/plain"] = np.stack(plain)
        out[name + "/default"] = np.stack(dflt)
        out[name + "/sums"] = np.stack(sums)
    path = os.path.join(ROOT, "tests", "golden", "text_crop_ref.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
