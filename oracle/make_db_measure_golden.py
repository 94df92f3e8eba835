"""Generate tests/golden/db_measure_ref.npz with the REFERENCE's own QuadMeasurer and DetectionIoUEvaluator
(structure/measurers/quad_measurer.py, concern/icdar2015_eval/detection/iou.py, loaded unmodified through oracle/ref_loader),
shapely's Polygon bound to the restatement of oracle/db_measure_port.py.

    python -m oracle.make_db_measure_golden

One environment fix, as in tests/test_db_measure_cpu.py: measure()'s np.array(output[0]) raises on a ragged batch under
numpy >= 1.24, so the module's numpy is given an `array` that falls back to an object array of per-image arrays
(ragged_numpy).  Cases are seeded (tests/db_measure_cases.py).  Per case the file holds the inputs (gt quads, tags, detections
padded to the largest count) and, per image, the reference's counts, metrics, pairs, don't-care lists, iouMat and
evaluationLog, flattened with their lengths; and gather_measure's meters over the case."""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import db_measure_port as port  # noqa: E402
from tests.db_measure_cases import batch_case  # noqa: E402

CASES = [  # name, seed, N, H, W, gt range, det range, gt dtype, int32 detections
    ("mixed", 1, 4, 640, 640, (0, 20), (0, 40), np.float64, True),
    ("f32", 2, 3, 320, 480, (3, 15), (5, 30), np.float32, False),
    ("many", 3, 2, 576, 1024, (20, 30), (110, 140), np.float64, True),
    ("sparse", 4, 6, 256, 256, (0, 3), (0, 3), np.float64, True),
]


def ragged_numpy():
    """numpy, except that array() of a ragged list gives an object array of per-image arrays"""
    shim = types.ModuleType("numpy_ragged")
    shim.__dict__.update(np.__dict__)

    def array(a, *args, **kw):
        try:
            return np.array(a, *args, **kw)
        except ValueError:
            out = np.empty(len(a), dtype=object)
            for i, x in enumerate(a):
                out[i] = np.array(x)
            return out
    shim.array = array
    return shim


def reference_measurer():
    from oracle import ref_loader
    if not ref_loader.install():
        return None
    iou = ref_loader.load("concern.icdar2015_eval.detection.iou")
    iou.Polygon = port.Polygon
    qm = ref_loader.load("structure.measurers.quad_measurer")
    qm.np = ragged_numpy()
    return qm.QuadMeasurer()


def case_inputs(seed, N, H, W, gt_range, det_range, gt_dtype, int_dets):
    images = batch_case(seed, N, H, W, gt_range, det_range, gt_dtype, int_dets)
    batch = dict(polygons=[g for g, _, _ in images], ignore_tags=[t for _, t, _ in images], image=np.zeros((N, 3, H, W)))
    boxes = [d.astype(np.float64).tolist() for _, _, d in images]          # as represent() gives them
    return batch, boxes


def main():
    m = reference_measurer()
    if m is None:
        raise SystemExit("reference tree not present")
    out = {}
    for name, seed, N, H, W, gr, dr, dt, idet in CASES:
        batch, boxes = case_inputs(seed, N, H, W, gr, dr, dt, idet)
        res = m.measure(batch, (boxes,))
        meters = m.gather_measure([res], None)
        maxd = max(len(b) for b in boxes)
        dets = np.zeros((N, maxd, 4, 2), np.float64)
        for n, b in enumerate(boxes):
            if b:
                dets[n, :len(b)] = b
        p = lambda k: [r[k] for r in res]  # noqa: E731
        out[name + "/gt"] = np.concatenate([np.asarray(g).reshape(-1, 4, 2) for g in batch['polygons']])
        out[name + "/gt_counts"] = np.array([len(g) for g in batch['polygons']])
        out[name + "/tags"] = np.concatenate(batch['ignore_tags']).astype(bool)
        out[name + "/dets"] = dets
        out[name + "/det_counts"] = np.array([len(b) for b in boxes])
        out[name + "/counts"] = np.array([[r['gtCare'], r['detCare'], r['detMatched']] for r in res])
        out[name + "/metrics"] = np.array([[r['precision'], r['recall'], r['hmean']] for r in res], np.float64)
        for key, src in (("pairs", [[(q['gt'], q['det']) for q in r['pairs']] for r in res]), ("gt_dc", p('gtDontCare')),
                         ("det_dc", p('detDontCare'))):
            out[name + "/" + key] = np.array([v for lst in src for v in lst], np.int64).reshape((-1, 2) if key == "pairs" else -1)
            out[name + "/" + key + "_len"] = np.array([len(lst) for lst in src])
        shapes = [np.asarray(r['iouMat']).shape if len(r['gtPolPoints']) and len(r['detPolPoints']) and r['iouMat'] != []
                  else (0, 0) for r in res]
        out[name + "/iou_shape"] = np.array([s if len(s) == 2 else (0, 0) for s in shapes])
        out[name + "/iou"] = np.concatenate([np.asarray(r['iouMat'], np.float64).reshape(-1) if s != (0, 0) else np.zeros(0)
                                             for r, s in zip(res, shapes)])
        out[name + "/log"] = np.array(p('evaluationLog'))
        out[name + "/meters"] = np.array([[getattr(meters[k], a) for a in ("val", "avg", "sum", "count")]
                                          for k in ("precision", "recall", "fmeasure")], np.float64)
    path = os.path.join(ROOT, "tests", "golden", "db_measure_ref.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
