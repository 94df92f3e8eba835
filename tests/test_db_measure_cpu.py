"""CPU: the PRODUCT's geometry of the DB validation measure (megreader_b200/csrc/db_measure_core.cuh -- the code the CUDA kernels
of csrc/db_measure.cu run) compiled for the host by tests/host_harness/db_measure_core_host.cpp, checked against
  * the exact oracle (oracle/db_measure_port.py) on about 20,000 seeded (gt, det) pairs and the hand pairs of
    tests/db_measure_cases.py: validity equal, IoU and intersection / area(det) within 1e-9 and bit-exact on axis-aligned
    integer boxes, every `> 0.5` decision equal;
  * a hand table of validity verdicts, one row per rule;
  * evaluate_image's metric arithmetic, bit for bit;
and the oracle against the reference's own iou.py and quad_measurer.py, run on the oracle's Polygon (skipped where the
reference tree is absent), including the reference raising on a ragged batch under the installed numpy."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import db_measure_port as port
from tests.db_measure_cases import batch_case, hand_pairs, pair_corpus

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("harness") / "libdb_measure_core_host.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                           "-I", os.path.join(HERE, "..", "megreader_b200", "csrc"),
                           os.path.join(HERE, "host_harness", "db_measure_core_host.cpp"), "-o", so])
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def host_pairs(lib, gt, det):
    gt, det = np.ascontiguousarray(gt, np.float64), np.ascontiguousarray(det, np.float64)
    n = len(gt)
    vg, vd = np.zeros(n, np.int32), np.zeros(n, np.int32)
    iou, prec = np.zeros(n), np.zeros(n)
    lib.host_pairs(_p(gt), _p(det), n, _p(vg), _p(vd), _p(iou), _p(prec))
    return vg.astype(bool), vd.astype(bool), iou, prec


def axis_aligned_integer(q):
    q = np.asarray(q)
    if not (q == np.round(q)).all():
        return False
    e = np.roll(q, -1, 0) - q
    return bool(((e[:, 0] == 0) | (e[:, 1] == 0)).all())


def test_core_equals_exact_oracle(harness):
    gt, det = pair_corpus(np.random.default_rng(5), 20000)
    hand = hand_pairs()
    gt = np.concatenate([gt, [g for _, g, _ in hand]])
    det = np.concatenate([det, [d for _, _, d in hand]])
    vg, vd, iou, prec = host_pairs(harness, gt, det)
    counts = dict(pairs=0, aligned=0, overlapping=0, ties=0)
    for i in range(len(gt)):
        pg, pd = port.Polygon(gt[i]), port.Polygon(det[i])
        assert (pg.is_valid, pd.is_valid) == (vg[i], vd[i]), (gt[i].tolist(), det[i].tolist())
        if not (vg[i] and vd[i]):
            continue
        counts["pairs"] += 1
        inter = pd.exact_intersection(pg)
        want_iou = float(inter) / pd.union(pg).area if inter else 0.0
        want_prec = float(pg.exact_intersection(pd)) / pd.area
        counts["overlapping"] += inter > 0
        if axis_aligned_integer(gt[i]) and axis_aligned_integer(det[i]):
            counts["aligned"] += 1
            assert (iou[i], prec[i]) == (want_iou, want_prec), (gt[i].tolist(), det[i].tolist())
        assert abs(iou[i] - want_iou) <= 1e-9 and abs(prec[i] - want_prec) <= 1e-9, (gt[i].tolist(), det[i].tolist())
        for got, want, exact in ((iou[i], want_iou, inter / (pd.exact_area() + pg.exact_area() - inter)),
                                 (prec[i], want_prec, inter / pd.exact_area())):
            if (got > 0.5) != (want > 0.5):
                # only where the exact value is within 1e-9 of the threshold, and in this corpus only at exact ties
                assert abs(exact - 0.5) <= 1e-9 and exact == 0.5, (gt[i].tolist(), det[i].tolist())
                counts["ties"] += 1
    assert counts["pairs"] > 15000 and counts["overlapping"] > 10000 and counts["aligned"] > 3000, counts
    assert counts["ties"] == 0, counts


def test_hand_pairs(harness):
    hand = hand_pairs()
    vg, vd, iou, prec = host_pairs(harness, [g for _, g, _ in hand], [d for _, _, d in hand])
    got = {name: (a, b, c, d) for (name, _, _), a, b, c, d in zip(hand, vg, vd, iou, prec)}
    assert got["identical"][2:] == (1.0, 1.0)
    assert got["contained"][2:] == (0.04, 1.0)
    assert got["disjoint"][2:] == got["edge_touch"][2:] == got["corner_touch"][2:] == (0.0, 0.0)
    ties = [(name, c, d) for (name, _, _), c, d in zip(hand, iou, prec) if name.endswith("_exact_tie")]
    assert all((c == 0.5) if name.startswith("iou") else (d == 0.5) for name, c, d in ties) and len(ties) == 4
    assert got["iou_plus_px"][2] > 0.5 > got["iou_minus_px"][2]
    assert not got["bow_tie"][0] and not got["sliver_line"][0]


# one row per validity rule of GEOS IsValidOp on one ring, and the valid shapes next to them
VALIDITY = [
    ("square", [[0, 0], [10, 0], [10, 10], [0, 10]], True),
    ("bow_tie", [[0, 0], [10, 10], [10, 0], [0, 10]], False),                 # non-adjacent edges cross
    ("vertex_on_edge", [[0, 0], [10, 0], [5, 0], [5, 5]], False),             # adjacent edges overlap (fold back)
    ("two_distinct_points", [[0, 0], [5, 5], [5, 5], [0, 0]], False),
    ("one_point", [[3, 3]] * 4, False),
    ("three_collinear", [[0, 0], [5, 5], [10, 10], [10, 10]], False),         # zero area
    ("spike", [[0, 0], [10, 0], [10, 10], [10, 5]], False),                   # fold-back at the last vertex
    ("touching_vertex", [[0, 0], [10, 0], [0, 10], [10, 0]], False),          # a vertex repeated, not consecutively
    ("collinear_middle_vertex", [[0, 0], [5, 0], [10, 0], [5, 8]], True),
    ("duplicate_corner_triangle", [[0, 0], [10, 0], [10, 0], [0, 10]], True),
    ("duplicate_first_last", [[0, 0], [10, 0], [0, 10], [0, 0]], True),
    ("concave_dart", [[0, 0], [5, 2], [10, 0], [5, 8]], True),
    ("clockwise", [[0, 0], [0, 10], [10, 10], [10, 0]], True),
    ("not_finite", [[0, 0], [np.nan, 0], [10, 10], [0, 10]], False),
    ("infinite", [[0, 0], [np.inf, 0], [10, 10], [0, 10]], False),
    ("thin_rectangle", [[0, 0], [2, 0], [2, 2 ** -40], [0, 2 ** -40]], True),
    ("nearly_collinear", [[0, 0], [1, 1], [2, 2 + 2 ** -51], [0, 3]], True),      # a turn of 2^-51 at (1, 1)
    ("collinear_fold_tiny", [[1, 1], [0, 0], [1e-300, 1e-300], [2, 3]], False),  # folds back at (0, 0)
]


@pytest.mark.parametrize("name,quad,valid", VALIDITY, ids=[v[0] for v in VALIDITY])
def test_validity_table(harness, name, quad, valid):
    q = np.ascontiguousarray(np.array(quad, np.float64).reshape(1, 4, 2))
    out = np.zeros(1, np.int32)
    harness.host_valid(_p(q), 1, _p(out))
    assert bool(out[0]) == valid
    assert port.Polygon(q[0]).is_valid == valid and port.Polygon(q[0]).is_simple == valid


def test_metrics_bit_equal(harness):
    out = np.zeros(3)
    for gt_care in range(0, 12):
        for det_care in range(0, 12):
            for matched in range(0, min(gt_care, det_care) + 1):
                harness.host_metrics(gt_care, det_care, matched, _p(out))
                if gt_care == 0:
                    r, p = float(1), float(0) if det_care > 0 else float(1)
                else:
                    r, p = float(matched) / gt_care, 0 if det_care == 0 else float(matched) / det_care
                h = 0 if (p + r) == 0 else 2.0 * p * r / (p + r)
                assert out.tolist() == [p, r, h]


# ---- the oracle against the reference's own evaluator and measurer ----

@pytest.fixture(scope="module")
def reference():
    from oracle import make_db_measure_golden as gen
    m = gen.reference_measurer()
    if m is None:
        pytest.skip("reference tree not present")
    import sys
    return m, sys.modules["structure.measurers.quad_measurer"], gen


def same_result(a, b, check_iou=True):
    assert a.keys() == b.keys()
    for k in a:
        if k in ("gtPolPoints", "detPolPoints"):
            assert len(a[k]) == len(b[k]) and all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a[k], b[k])), k
        elif k == "iouMat":
            if check_iou:
                assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
        else:
            assert a[k] == b[k] and type(a[k]) is type(b[k]), (k, a[k], b[k])


@pytest.mark.parametrize("seed,gt_dtype,int_dets", [(11, np.float64, True), (12, np.float32, False), (13, np.float64, False)])
def test_oracle_equals_reference(reference, seed, gt_dtype, int_dets):
    m, _, gen = reference
    batch, boxes = gen.case_inputs(seed, 5, 320, 320, (0, 12), (0, 25), gt_dtype, int_dets)
    want = m.measure(batch, (boxes,))
    got = port.QuadMeasurer().measure(batch, (boxes,))
    for w, g in zip(want, got):
        # np.empty([1, 1]) is uninitialised in the reference; the restatement gives [[0.0]]
        same_result(w, g, check_iou=bool(w['gtPolPoints']) and bool(w['detPolPoints']))
    mw, mg = m.gather_measure([want, want[:2]], None), port.QuadMeasurer().gather_measure([got, got[:2]])
    for k in ("precision", "recall", "fmeasure"):
        assert [getattr(mw[k], a) for a in ("val", "avg", "sum", "count")] == [getattr(mg[k], a) for a in ("val", "avg", "sum", "count")]


def test_reference_raises_on_ragged_batch(reference, monkeypatch):
    m, qm, gen = reference
    batch, boxes = gen.case_inputs(14, 2, 128, 128, (1, 3), (1, 3), np.float64, True)
    boxes = [boxes[0], boxes[0] + boxes[0]]            # two images with different box counts
    monkeypatch.setattr(qm, "np", np)                 # the installed numpy, unpatched
    with pytest.raises(ValueError, match="inhomogeneous"):
        m.measure(batch, (boxes,))


def test_golden_is_current(reference):
    """the committed golden equals what the generator makes now from the reference"""
    _, _, gen = reference
    z = np.load(os.path.join(HERE, "golden", "db_measure_ref.npz"))
    for name, seed, N, H, W, gr, dr, dt, idet in gen.CASES:
        images = batch_case(seed, N, H, W, gr, dr, dt, idet)
        assert np.array_equal(z[name + "/gt"], np.concatenate([g.reshape(-1, 4, 2) for g, _, _ in images]))
        assert z[name + "/det_counts"].tolist() == [len(d) for _, _, d in images]


# ---- construction as the yaml's config builds it ----

def test_quad_measurer_takes_config_keywords():
    """concern/config.py builds `measurer: class: ...` as cls(**args, cmd=cmd) with `class` still in args"""
    from megreader_b200 import db_measure
    m = db_measure.QuadMeasurer(**{'class': 'structure.measurers.QuadMeasurer'}, cmd={})
    assert (m.iou_constraint, m.area_precision_constraint, m.device) == (0.5, 0.5, None)


def test_quad_measurer_built_by_reference_config():
    """the reference's own create_member_from_config builds the delegated class (skipped where the reference is absent)"""
    from oracle import ref_loader
    if not ref_loader.install():
        pytest.skip("reference tree not present")
    config = ref_loader.load("concern.config")
    builder = config.Configurable.create_member_from_config
    m = builder(config.Configurable, ({'class': 'megreader_b200.db_measure.QuadMeasurer'}, {'name': 'x'}))
    from megreader_b200 import db_measure
    assert type(m) is db_measure.QuadMeasurer and m.iou_constraint == 0.5
