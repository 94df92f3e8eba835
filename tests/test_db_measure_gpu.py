"""GPU: the DB validation measure (megreader_b200.db_measure, csrc/db_measure.cu) against
  * the golden recorded from the reference's own QuadMeasurer / DetectionIoUEvaluator (tests/golden/db_measure_ref.npz);
  * the live oracle (oracle/db_measure_port.py) on bigger batches with float32 and float64 gt, and at the yaml's validation
    shape with detections from boxes_from_maps and gt from make_targets_packed;
and its QuadMeasurer structures, edge cases, refusals and CUDA graph capture, alone and in the whole validation step."""
import os

import numpy as np
import pytest
import torch

from oracle import db_measure_port as port
from tests.db_measure_cases import batch_case

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("CUDA not available")
    return torch.device("cuda")


def packed(images, dev, capacity=None, maxd=None):
    """per-image (gt, tags, dets) -> the packed device inputs of evaluate_packed"""
    from megreader_b200 import db_targets
    polys, tags, offsets = db_targets.pack([torch.from_numpy(np.ascontiguousarray(g)).to(dev) for g, _, _ in images],
                                           [torch.from_numpy(t).to(dev) for _, t, _ in images], capacity)
    maxd = max([len(d) for _, _, d in images] + [0]) if maxd is None else maxd
    ddt = images[0][2].dtype if images else np.float64
    boxes = np.zeros((len(images), maxd, 4, 2), ddt)
    for n, (_, _, d) in enumerate(images):
        boxes[n, :len(d)] = d
    count = torch.tensor([len(d) for _, _, d in images], dtype=torch.int32).to(dev)
    return polys, tags, offsets, torch.from_numpy(boxes).to(dev), count


def decode(out, offsets, tags):
    """per image, from the device's outputs and the gt tags: pairs, gtDontCare, detDontCare, (gtCare, detCare, detMatched),
    metrics, iou among valid polygons"""
    h = {k: v.cpu().numpy() for k, v in out.items() if torch.is_tensor(v) and k != "workspace"}
    off, tg = offsets.cpu().numpy(), tags.cpu().numpy()
    res = []
    for n in range(len(off) - 1):
        gi, gm, gt = h["gt_index"][off[n]:off[n + 1]], h["gt_match"][off[n]:off[n + 1]], tg[off[n]:off[n + 1]]
        di = h["det_index"][n]
        gv, dv = np.nonzero(gi >= 0)[0], np.nonzero(di >= 0)[0]
        r = dict(pairs=[(int(gi[k]), int(gm[k])) for k in gv if gm[k] >= 0], gt_dc=[int(gi[k]) for k in gv if gt[k]],
                 det_dc=[int(di[j]) for j in dv if h["det_dontcare"][n, j]],
                 counts=tuple(int(v) for v in h["counts"][n, :3]), valid=(len(gv), len(dv)),
                 metrics=tuple(float(v) for v in h["metrics"][n]), status=int(h["status"][n]))
        if "iou" in h:
            r["iou"] = h["iou"][off[n] + gv][:, dv]
        res.append(r)
    return res


def oracle_images(images):
    return [port.evaluate_image([dict(points=g[i], ignore=bool(t[i])) for i in range(len(g))],
                                [dict(points=d[i]) for i in range(len(d))]) for g, t, d in images]


def assert_matches_oracle(got, want, check_iou=True):
    for n, (g, w) in enumerate(zip(got, want)):
        assert g["status"] == 0
        assert g["pairs"] == [(p['gt'], p['det']) for p in w['pairs']], n
        assert g["det_dc"] == w['detDontCare'], n
        assert g["gt_dc"] == w['gtDontCare'], n
        assert g["counts"] == (w['gtCare'], w['detCare'], w['detMatched']), n
        assert g["valid"] == (len(w['gtPolPoints']), len(w['detPolPoints'])), n
        assert g["metrics"] == (w['precision'], w['recall'], w['hmean']), n
        if check_iou and w['iouMat'] != [] and g["valid"][0] and g["valid"][1]:
            np.testing.assert_allclose(g["iou"], np.asarray(w['iouMat']), rtol=0, atol=1e-9)


def test_golden():
    from megreader_b200 import db_measure
    dev = _dev()
    z = np.load(os.path.join(HERE, "golden", "db_measure_ref.npz"))
    for name in ("mixed", "f32", "many", "sparse"):
        gc, dc = z[name + "/gt_counts"], z[name + "/det_counts"]
        go = np.concatenate([[0], np.cumsum(gc)])
        images = [(z[name + "/gt"][go[n]:go[n + 1]], z[name + "/tags"][go[n]:go[n + 1]], z[name + "/dets"][n, :dc[n]])
                  for n in range(len(gc))]
        polys, tags, offsets, boxes, count = packed(images, dev)
        totals = torch.zeros(3, dtype=torch.int64, device=dev)
        got = decode(db_measure.evaluate_packed(polys, tags, offsets, boxes, count, totals=totals, with_iou=True), offsets, tags)
        split = lambda key, lens: np.split(z[name + "/" + key], np.cumsum(lens)[:-1])  # noqa: E731
        pairs, gdc, ddc = split("pairs", z[name + "/pairs_len"]), split("gt_dc", z[name + "/gt_dc_len"]), split("det_dc", z[name + "/det_dc_len"])
        shapes = z[name + "/iou_shape"]
        ious = split("iou", [int(a) * int(b) for a, b in shapes])
        for n, g in enumerate(got):
            assert g["status"] == 0
            assert g["pairs"] == [tuple(p) for p in pairs[n].tolist()], (name, n)
            assert g["det_dc"] == ddc[n].tolist(), (name, n)
            assert g["gt_dc"] == gdc[n].tolist(), (name, n)
            assert g["counts"] == tuple(z[name + "/counts"][n].tolist()), (name, n)
            assert g["metrics"] == tuple(z[name + "/metrics"][n].tolist()), (name, n)
            if shapes[n][0]:
                np.testing.assert_allclose(g["iou"], ious[n].reshape(shapes[n]), rtol=0, atol=1e-9)
        c = z[name + "/counts"].sum(0)
        assert totals.tolist() == c.tolist()
        m = db_measure.combine(totals)
        meters = z[name + "/meters"]
        assert m['precision'] == meters[0, 0] and m['recall'] == meters[1, 0]
        # QuadMeasurer on the same case: the log strings and gather_measure's meters, bit for bit
        qm = db_measure.QuadMeasurer()
        batch = dict(polygons=[g for g, _, _ in images], ignore_tags=[t for _, t, _ in images])
        res = qm.measure(batch, ([d.tolist() for _, _, d in images],))
        assert [r['evaluationLog'] for r in res] == z[name + "/log"].tolist()
        mt = qm.gather_measure([res], None)
        assert [[getattr(mt[k], a) for a in ("val", "avg", "sum", "count")] for k in ("precision", "recall", "fmeasure")] \
            == meters.tolist()


@pytest.mark.parametrize("gt_dtype", [np.float64, np.float32])
def test_live_oracle_big_batch(gt_dtype):
    from megreader_b200 import db_measure
    dev = _dev()
    images = batch_case(21 + (gt_dtype == np.float32), 16, 640, 640, (0, 100), (0, 1000), gt_dtype, True, noise=0.5)
    polys, tags, offsets, boxes, count = packed(images, dev)
    assert boxes.size(1) > 500 and max(len(g) for g, _, _ in images) > 50
    got = decode(db_measure.evaluate_packed(polys, tags, offsets, boxes, count, with_iou=True), offsets, tags)
    want = oracle_images(images)
    assert_matches_oracle(got, want)
    assert sum(g["counts"][2] for g in got) > 100


def test_live_oracle_float_dets():
    from megreader_b200 import db_measure
    dev = _dev()
    images = batch_case(23, 6, 480, 480, (0, 40), (0, 80), np.float64, False, odd=0.4)
    polys, tags, offsets, boxes, count = packed(images, dev)
    got = decode(db_measure.evaluate_packed(polys, tags, offsets, boxes, count, with_iou=True), offsets, tags)
    assert_matches_oracle(got, oracle_images(images))


def render_maps(images, H, W, dev, seed):
    """gt quads -> make_targets_packed (validated gt, updated tags, shrunk text map) -> a noisy probability map"""
    from megreader_b200 import db_targets
    polys, tags, offsets = db_targets.pack([torch.from_numpy(g).to(dev) for g, _, _ in images],
                                           [torch.from_numpy(t).to(dev) for _, t, _ in images])
    t = db_targets.make_targets_packed(polys, tags, offsets, (H, W))
    gen = torch.Generator(device=dev).manual_seed(seed)
    prob = (t["gt"] * 0.9 + 0.15 * torch.rand(t["gt"].shape, generator=gen, device=dev)).clamp(0, 1)
    return t, offsets, prob


@pytest.mark.parametrize("gt_dtype", [np.float64, np.float32])
def test_yaml_validation_shape(gt_dtype):
    """4 x 576 x 1024: maps rendered from the gt, boxes_from_maps(max_candidates=1000), make_targets_packed, evaluate_packed"""
    from megreader_b200 import db_boxes, db_measure
    dev = _dev()
    H, W = 576, 1024
    images = batch_case(31, 4, H, W, (20, 40), (0, 0), gt_dtype)
    t, offsets, prob = render_maps(images, H, W, dev, 5)
    boxes, _, count = db_boxes.boxes_from_maps(prob, None, 0.3, 0.7, 1000)
    out = db_measure.evaluate_packed(t["polygons"], t["ignore_tags"], offsets, boxes, count, with_iou=True)
    got = decode(out, offsets, t["ignore_tags"])
    off = offsets.cpu().numpy()
    vp, vt, bx, cn = t["polygons"].cpu().numpy(), t["ignore_tags"].cpu().numpy().astype(bool), boxes.cpu().numpy(), count.cpu().numpy()
    host = [(vp[off[n]:off[n + 1]], vt[off[n]:off[n + 1]], bx[n, :cn[n]]) for n in range(4)]
    assert_matches_oracle(got, oracle_images(host))
    # most detections are text the maps were rendered from (touching boxes merge into one contour, so not every gt is found)
    matched = sum(g["counts"][2] for g in got)
    assert sum(g["valid"][1] for g in got) > 30 and matched > 0.5 * sum(g["counts"][1] for g in got)


def test_quad_measurer_structures():
    from megreader_b200 import db_measure
    _dev()
    images = batch_case(41, 5, 320, 320, (0, 12), (0, 25), np.float32, False)
    images[1] = (images[1][0][:0], images[1][1][:0], images[1][2])            # no gt
    images[2] = (images[2][0], images[2][1], images[2][2][:0])                 # no dets
    batch = dict(polygons=[g for g, _, _ in images], ignore_tags=[t for _, t, _ in images], image=np.zeros((5, 3, 8, 8)))
    boxes = [d.tolist() for _, _, d in images]
    qm, ref = db_measure.QuadMeasurer(), port.QuadMeasurer()
    got, want = qm.validate_measure(batch, (boxes,)), ref.validate_measure(batch, (boxes,))
    assert got[1] == want[1] == [0]
    for g, w in zip(got[0], want[0]):
        assert g.keys() == w.keys()
        for k in g:
            if k in ("gtPolPoints", "detPolPoints"):
                assert len(g[k]) == len(w[k]) and all(np.array_equal(a, np.asarray(b)) for a, b in zip(g[k], w[k]))
            elif k == "iouMat":
                np.testing.assert_allclose(np.asarray(g[k]), np.asarray(w[k]), rtol=0, atol=1e-9)
                assert np.asarray(g[k]).shape == np.asarray(w[k]).shape
            else:
                assert g[k] == w[k] and type(g[k]) is type(w[k]), (k, g[k], w[k])
    mg, mw = qm.gather_measure([got[0], got[0][:3]], None), ref.gather_measure([want[0], want[0][:3]])
    for k in ("precision", "recall", "fmeasure"):
        assert [getattr(mg[k], a) for a in ("val", "avg", "sum", "count")] == [getattr(mw[k], a) for a in ("val", "avg", "sum", "count")]
    # the tensors of boxes_from_maps give the same results as represent()'s lists
    dev = torch.device("cuda")
    _, _, _, bt, ct = packed([(g, t, d.astype(np.int32)) for g, t, d in batch_case(42, 3, 320, 320, (1, 8), (1, 12))], dev)
    lists = [bt[n, :int(ct[n])].cpu().numpy().astype(np.float64).tolist() for n in range(3)]
    b2 = dict(polygons=[g for g, _, _ in batch_case(42, 3, 320, 320, (1, 8), (1, 12))],
              ignore_tags=[t for _, t, _ in batch_case(42, 3, 320, 320, (1, 8), (1, 12))])
    a, b = qm.measure(b2, ((bt, None, ct),)), qm.measure(b2, (lists,))
    assert [r['pairs'] for r in a] == [r['pairs'] for r in b] and [r['evaluationLog'] for r in a] == [r['evaluationLog'] for r in b]
    with pytest.raises(ValueError, match="quads"):
        qm.measure(dict(polygons=[np.zeros((2, 5, 2))], ignore_tags=[np.zeros(2, bool)]), ([[]],))


def test_edge_cases():
    from megreader_b200 import db_measure
    dev = _dev()
    sq = lambda x, y, s: np.array([[x, y], [x + s, y], [x + s, y + s], [x, y + s]], np.float64)  # noqa: E731
    bow = np.array([[0, 0], [10, 10], [10, 0], [0, 10]], np.float64)
    images = [
        (np.zeros((0, 4, 2)), np.zeros(0, bool), np.array([sq(0, 0, 10)])),                       # no gt
        (np.array([sq(0, 0, 10)]), np.array([False]), np.zeros((0, 4, 2))),                       # no dets
        (np.array([sq(0, 0, 10), sq(20, 0, 10)]), np.array([True, True]), np.array([sq(0, 0, 9), sq(50, 50, 5)])),  # only don't care
        (np.array([bow, bow]), np.array([False, True]), np.array([bow, sq(0, 0, 0)])),            # only invalid polygons
        (np.zeros((0, 4, 2)), np.zeros(0, bool), np.zeros((0, 4, 2))),                            # nothing
    ]
    polys, tags, offsets, boxes, count = packed(images, dev)
    totals = torch.zeros(3, dtype=torch.int64, device=dev)
    got = decode(db_measure.evaluate_packed(polys, tags, offsets, boxes, count, totals=totals, with_iou=True), offsets, tags)
    assert_matches_oracle(got, oracle_images(images))
    assert got[2]["det_dc"] == [0] and got[3]["valid"] == (0, 0)
    assert totals.tolist() == [sum(g["counts"][k] for g in got) for k in range(3)]
    # max_dets = 0
    polys, tags, offsets, boxes, count = packed([(g, t, d[:0]) for g, t, d in images], dev)
    assert boxes.size(1) == 0
    got = decode(db_measure.evaluate_packed(polys, tags, offsets, boxes, count), offsets, tags)
    assert_matches_oracle(got, oracle_images([(g, t, d[:0]) for g, t, d in images]), check_iou=False)


def test_slots_outside_the_offsets():
    """gt slots before offsets[0] and from offsets[N] on belong to no image: a don't-care quad there that covers image 0's
    detections neither marks them don't-care nor gets an index"""
    from megreader_b200 import db_measure
    dev = _dev()
    images = batch_case(55, 3, 300, 300, (3, 8), (3, 10))
    polys, tags, offsets, boxes, count = packed(images, dev)
    cover = torch.tensor([[-1, -1], [400, -1], [400, 400], [-1, 400]], dtype=polys.dtype, device=dev).reshape(1, 4, 2)
    polys2 = torch.cat([cover, polys, cover])
    tags2 = torch.cat([torch.ones(1, dtype=torch.uint8, device=dev), tags, torch.ones(1, dtype=torch.uint8, device=dev)])
    out = db_measure.evaluate_packed(polys2, tags2, offsets + 1, boxes, count, with_iou=True)
    assert out["gt_index"][0].item() == -1 and out["gt_index"][-1].item() == -1
    assert out["status"].tolist() == [0, 0, 0]
    got = decode(out, offsets + 1, tags2)
    assert_matches_oracle(got, oracle_images(images))
    assert not out["iou"][0].any() and not out["iou"][-1].any()


def test_refusals():
    from megreader_b200 import db_measure
    dev = _dev()
    images = batch_case(51, 3, 200, 200, (2, 5), (2, 5))
    polys, tags, offsets, boxes, count = packed(images, dev)
    with pytest.raises(NotImplementedError):
        db_measure.evaluate_packed(polys.cpu(), tags, offsets, boxes, count)
    with pytest.raises(NotImplementedError):
        db_measure.evaluate_packed(polys, tags, offsets, boxes.cpu(), count)
    with pytest.raises(RuntimeError):
        db_measure.evaluate_packed(polys.half(), tags, offsets, boxes, count)
    with pytest.raises(RuntimeError):
        db_measure.evaluate_packed(polys, tags, offsets, boxes.float(), count)
    with pytest.raises(RuntimeError):
        db_measure.evaluate_packed(polys, tags.bool(), offsets, boxes, count)
    with pytest.raises(RuntimeError):
        db_measure.evaluate_packed(polys, tags, offsets.long(), boxes, count)
    with pytest.raises(RuntimeError):
        db_measure.evaluate_packed(polys, tags, offsets, boxes[:2], count)
    with pytest.raises(RuntimeError):
        db_measure.evaluate_packed(polys, tags, offsets, boxes, count[:2])
    with pytest.raises(RuntimeError):
        db_measure.evaluate_packed(polys, tags, offsets, boxes, count, totals=torch.zeros(3, dtype=torch.int32, device=dev))
    # bad device contents: reported per image, never a fault, and kept out of the totals
    totals = torch.zeros(3, dtype=torch.int64, device=dev)
    bad_count = count.clone()
    bad_count[1] = boxes.size(1) + 5
    bad_off = offsets.clone()
    bad_off[2] = polys.size(0) + 7
    out = db_measure.evaluate_packed(polys, tags, bad_off, boxes, bad_count, totals=totals)
    st = out["status"].tolist()
    assert st[0] == 0 and st[1] & db_measure.BAD_COUNT and st[1] & db_measure.BAD_OFFSETS and st[2] & db_measure.BAD_OFFSETS
    assert totals.tolist() == out["counts"][0, :3].tolist()
    torch.cuda.synchronize()


def test_graph_capture_totals():
    from megreader_b200 import db_measure
    dev = _dev()
    batches = [batch_case(60 + k, 4, 400, 400, (0, 30), (0, 60), np.float32) for k in range(3)]
    cap = max(sum(len(g) for g, _, _ in b) for b in batches)
    maxd = max(len(d) for b in batches for _, _, d in b)
    inputs = [packed(b, dev, cap, maxd) for b in batches]
    eager = torch.zeros(3, dtype=torch.int64, device=dev)
    eager_out = [db_measure.evaluate_packed(*x, totals=eager) for x in inputs]
    static = [t.clone() for t in inputs[0]]
    totals = torch.zeros(3, dtype=torch.int64, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        db_measure.evaluate_packed(*static)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = db_measure.evaluate_packed(*static, totals=totals)
    totals.zero_()
    for k, x in enumerate(inputs):
        for a, b in zip(static, x):
            a.copy_(b)
        g.replay()
        for key in ("counts", "metrics", "gt_match", "det_match", "det_dontcare"):
            assert torch.equal(out[key], eager_out[k][key]), (k, key)
    torch.cuda.synchronize()
    assert totals.tolist() == eager.tolist() and totals[0] > 0
    assert db_measure.combine(totals) == db_measure.combine(eager.cpu())


def test_validation_step_in_one_graph():
    """seg_detector_db.yaml's eval model on the engine convolutions, boxes_from_maps, make_targets_packed and evaluate_packed:
    one CUDA graph adding into device totals, replayed on a second batch, equal to the eager run"""
    import bench_trunks
    from megreader_b200 import db_boxes, db_measure, db_targets
    dev = _dev()
    torch.manual_seed(0)
    net, _ = bench_trunks.build(6, dev, engine=True)
    net.eval()
    H = W = 256
    x1, _ = bench_trunks.synth_db(2, 2, (H, W))
    x2, _ = bench_trunks.synth_db(3, 2, (H, W))
    x1, x2 = x1.to(dev), x2.to(dev)
    gts = [batch_case(70 + k, 2, H, W, (3, 8), (0, 0)) for k in range(2)]
    cap = max(sum(len(g) for g, _, _ in b) for b in gts)
    packs = [db_targets.pack([torch.from_numpy(g).to(dev) for g, _, _ in b], [torch.from_numpy(t).to(dev) for _, t, _ in b], cap)
             for b in gts]

    def step(x, polys, tags, offsets, totals):
        binary = net.decoder(net.backbone(x))
        binary = binary['binary'] if isinstance(binary, dict) else binary
        boxes, _, count = db_boxes.boxes_from_maps(binary.float(), None, 0.3, 0.5, 1000)
        t = db_targets.make_targets_packed(polys, tags, offsets, (H, W))
        return db_measure.evaluate_packed(t["polygons"], t["ignore_tags"], offsets, boxes, count, totals=totals)

    with torch.no_grad():
        eager_totals = torch.zeros(3, dtype=torch.int64, device=dev)
        eager = step(x2, *packs[1], eager_totals)
        static = [x1.clone()] + [t.clone() for t in packs[0]]
        totals = torch.zeros(3, dtype=torch.int64, device=dev)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step(*static, torch.zeros(3, dtype=torch.int64, device=dev))
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = step(*static, totals)
        static[0].copy_(x2)
        for a, b in zip(static[1:], packs[1]):
            a.copy_(b)
        totals.zero_()
        g.replay()
        torch.cuda.synchronize()
    for key in ("counts", "metrics", "gt_match", "det_match", "det_dontcare", "status"):
        assert torch.equal(out[key], eager[key]), key
    assert totals.tolist() == eager_totals.tolist() and totals[0] > 0
