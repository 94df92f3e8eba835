"""GPU: the DB contour step on the device (megreader_b200/db_boxes.find_contours, csrc/db_boxes.cu) against
cv2.findContours(RETR_LIST, CHAIN_APPROX_NONE)[:max_candidates] (seg_detector_representer.py:60-80) -- live where cv2 is importable,
else against tests/golden/db_contours_ref.npz -- contour for contour and point for point, at the yaml's validation shape and odd
sizes, with limits below and above the number of contours; get_mini_boxes and box_score_fast (:80-94, 125-168) of every kept
contour (db_boxes.box_candidates) against cv2.minAreaRect / cv2.boxPoints / cv2.fillPoly / cv2.mean; empty / full / all-hole maps,
repeatability and graph capture."""
import os

import numpy as np
import pytest
import torch

from tests.db_boxes_cases import BOX_GOLDEN_CASES, GPU_CASES, adversarial_bitmaps, case_maps, digest
from tests.make_db_contours_golden import bitmap_digest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "db_contours_ref.npz")

try:
    import cv2  # noqa: F401
    from tests.db_boxes_cases import box_score_fast, cv2_contours, reference_candidates
except ImportError:
    box_score_fast = cv2_contours = reference_candidates = None


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def run(maps, thresh, maxc, **kw):
    from megreader_b200 import db_boxes
    out = db_boxes.find_contours(torch.from_numpy(maps).to(_dev()), thresh, maxc, **kw)
    return out, db_boxes.contour_lists(*out[:3])


@pytest.mark.parametrize("name", [c[0] for c in GPU_CASES])
def test_contours_equal_reference(name):
    maps, thresh, maxc = case_maps(name)
    (points, offsets, count, total), got = run(maps, thresh, maxc)
    total = total.cpu().numpy()
    assert count.cpu().numpy().tolist() == np.minimum(total, maxc).tolist()
    if cv2_contours is not None:
        for n, m in enumerate(maps):
            want = cv2_contours(m[0] > np.float32(thresh))
            assert total[n] == len(want), n
            kept = want[:maxc]
            assert len(got[n]) == len(kept)
            for c, (g, w) in enumerate(zip(got[n], kept)):
                assert g.dtype == np.int32 and np.array_equal(g, w), (n, c)
    g = np.load(GOLD)
    assert list(g[name + ".bitmap"]) == bitmap_digest(maps, thresh), "the seeded maps differ from the ones the golden was made from"
    assert total.tolist() == g[name + ".total"].tolist()
    assert [digest(cs) for cs in got] == list(g[name + ".digest"])
    if name.startswith("val_"):
        assert (total > 1000).all()                  # both limits truncate


def assert_candidates_match(got, want, kept, maps):
    """bit for bit, except the class tests/test_db_boxes_cpu.py counts: a rectangle several hull edges give, where the calipers'
    float tie goes to another edge than cv2's -- the same box a few float ulps apart, on at most 0.2 % of the contours.  Its
    corners can truncate to another integer quad, so its score is checked against box_score_fast of the box it has."""
    boxes, ssides, scores = got
    want_boxes, want_ssides, want_scores = want
    same = (boxes == want_boxes).all(axis=(2, 3)) & (ssides == want_ssides)
    assert (scores[same] == want_scores[same]).all()
    for n, c in zip(*np.nonzero(~same)):
        tol = 4 * np.spacing(np.float32(max(np.abs(want_boxes[n, c]).max(), 1.0)))
        assert np.abs(boxes[n, c] - want_boxes[n, c]).max() <= tol, (n, c, boxes[n, c].tolist(), want_boxes[n, c].tolist())
        assert abs(ssides[n, c] - want_ssides[n, c]) <= tol, (n, c)
        if box_score_fast is not None and ssides[n, c] >= 3:
            assert scores[n, c] == box_score_fast(maps[n].reshape(maps.shape[-2:]), boxes[n, c]), (n, c)
    assert (~same).sum() <= max(2, 0.002 * kept), int((~same).sum())


def candidates(maps, thresh, maxc, **kw):
    from megreader_b200 import db_boxes
    x = torch.from_numpy(maps).to(_dev())
    points, offsets, count, total = db_boxes.find_contours(x, thresh, maxc, **kw)
    return (points, offsets, count, total), db_boxes.box_candidates(x, points, offsets, count)


@pytest.mark.parametrize("name", [c[0] for c in GPU_CASES])
def test_box_candidates_equal_reference(name):
    maps, thresh, maxc = case_maps(name)
    (_, _, count, _), got = candidates(maps, thresh, maxc)
    got = tuple(t.cpu().numpy() for t in got)
    if reference_candidates is not None:
        want = reference_candidates(maps, thresh, maxc)
    elif name in BOX_GOLDEN_CASES:
        g = np.load(GOLD)
        want = g[name + ".boxes"], g[name + ".ssides"], g[name + ".scores"]
    else:
        pytest.skip("needs cv2 for the reference candidates of this case")
    assert_candidates_match(got, want, int(count.sum()), maps)
    assert (got[2][got[1] < 3] == 0).all()


def test_small_point_capacity_is_reported():
    maps, thresh, _ = case_maps("odd_3x33x47")
    from megreader_b200 import db_boxes
    out = db_boxes.find_contours(torch.from_numpy(maps).to(_dev()), thresh, 1000, point_capacity=8)
    with pytest.raises(RuntimeError, match="point capacity"):
        db_boxes.contour_lists(*out[:3])
    _, ssides, _ = db_boxes.box_candidates(torch.from_numpy(maps).to(_dev()), *out[:3])
    off, cnt = out[1].cpu().numpy(), out[2].cpu().numpy()
    for n in range(len(cnt)):                            # contours that did not fit are flagged, the others are measured
        fits = off[n, 1:cnt[n] + 1] <= 8
        assert (ssides[n, :cnt[n]].cpu().numpy()[~fits] == -1).all() and (ssides[n, :cnt[n]].cpu().numpy()[fits] >= 0).all()


def test_empty_full_and_hole_maps():
    z = np.zeros((1, 1, 24, 40), np.float32)
    full = np.ones_like(z)
    holes = np.ones_like(z)
    holes[0, 0, 1:-1:2, 1:-1:2] = 0.0                 # every other interior pixel: 11 x 19 one-pixel holes
    maps = np.concatenate([z, full, holes])
    (_, _, count, total), got = run(maps, 0.5, 1000)
    assert total.tolist() == [0, 1, 1 + 11 * 19]
    assert got[0] == []
    border = got[1][0].reshape(-1, 2)
    assert len(border) == 2 * (24 + 40) - 4 and border[0].tolist() == [0, 0]
    assert {tuple(p) for p in border} == {(x, y) for y in range(24) for x in range(40) if x in (0, 39) or y in (0, 23)}
    if cv2_contours is not None:
        for n in range(3):
            want = cv2_contours(maps[n, 0] > 0.5)
            assert len(got[n]) == len(want) and all(np.array_equal(a, b) for a, b in zip(got[n], want))
    (_, _, count, total), got = run(holes, 0.5, 0)     # max_candidates = 0: nothing kept, the contours still counted
    assert count.tolist() == [0] and total.tolist() == [1 + 11 * 19] and got == [[]]


def test_adversarial_bitmaps_one_batch_each():
    if cv2_contours is None:
        pytest.skip("needs cv2 for the reference")
    for name, bm in sorted(adversarial_bitmaps().items()):
        _, got = run(bm[None, None].astype(np.float32), 0.5, 1000)
        want = cv2_contours(bm)
        assert len(got[0]) == len(want) and all(np.array_equal(a, b) for a, b in zip(got[0], want)), name


def test_repeatable_and_graph_capturable():
    from megreader_b200 import db_boxes
    dev = _dev()
    a, thresh, maxc = case_maps("val_4x576x1024_c1000")
    b = np.ascontiguousarray(a[::-1, :, :, ::-1])                     # another batch of the same shape
    xa, xb = torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)
    step = lambda x: (lambda o: o + db_boxes.box_candidates(x, *o[:3]))(db_boxes.find_contours(x, thresh, maxc))  # noqa: E731
    e1, e2, eb = step(xa), step(xa), step(xb)
    torch.cuda.synchronize()
    lists = lambda o: db_boxes.contour_lists(*o[:3])  # noqa: E731
    assert all(torch.equal(u, v) for u, v in zip(e1[1:], e2[1:]))
    assert [digest(x) for x in lists(e1)] == [digest(x) for x in lists(e2)]
    static = xa.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(static)                                                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gout = step(static)
    static.copy_(xb)
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(u, v) for u, v in zip(gout[1:], eb[1:]))
    assert [digest(x) for x in lists(gout)] == [digest(x) for x in lists(eb)]
    if cv2_contours is not None:
        want = [digest(cv2_contours(m[0] > np.float32(thresh))[:maxc]) for m in b]
        assert [digest(x) for x in lists(gout)] == want
