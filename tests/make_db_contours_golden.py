"""Writes tests/golden/db_contours_ref.npz: for every case of tests/db_boxes_cases.GPU_CASES and every image, the number of
contours cv2.findContours(RETR_LIST, CHAIN_APPROX_NONE) finds, the digest of the first max_candidates of them, and the digest of
the bitmap they came from (so that a GPU machine without cv2 can tell a changed input from a changed result); for the cases of
BOX_GOLDEN_CASES also the corners and ssides of get_mini_boxes and the box_score_fast scores (seg_detector_representer.py:80-94,
125-168) of every kept contour.

    python -m tests.make_db_contours_golden
"""
import hashlib
import os

import numpy as np

from tests.db_boxes_cases import BOX_GOLDEN_CASES, GPU_CASES, case_maps, reference, reference_candidates

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "db_contours_ref.npz")


def bitmap_digest(maps, thresh):
    return [hashlib.sha256(np.packbits(m > np.float32(thresh)).tobytes()).hexdigest() for m in maps]


def main():
    out = {}
    for name, *_ in GPU_CASES:
        maps, thresh, maxc = case_maps(name)
        ref = reference(maps, thresh, maxc)
        out[name + ".total"] = np.array([t for t, _ in ref], np.int64)
        out[name + ".digest"] = np.array([d for _, d in ref])
        out[name + ".bitmap"] = np.array(bitmap_digest(maps, thresh))
        if name in BOX_GOLDEN_CASES:
            out[name + ".boxes"], out[name + ".ssides"], out[name + ".scores"] = reference_candidates(maps, thresh, maxc)
    np.savez_compressed(OUT, **out)
    print(OUT)


if __name__ == "__main__":
    main()
