"""GPU: megreader_b200.text_crop (csrc/text_crop.cu) against the host harness of the same core (text_crop_core.cuh) bit for bit
on seeded ragged batches -- uint8 and float32 images, images without quads, int32 [N, K] boxes with counts and packed float32
quads with offsets, int32 boxes straight from boxes_from_maps, both modes -- the golden's cases, the row order, owner, total,
overflow, refusals, CUDA-graph replay, and the detection-to-strings chain captured as one graph."""
import numpy as np
import pytest
import torch

from megreader_b200 import _lib, db_batch, text_crop
from tests import text_crop_cases as C

pytestmark = pytest.mark.gpu

SHAPES = [(150, 230), (96, 128), (210, 170)]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    L = C.build_harness(tmp_path_factory.mktemp("harness"))
    if L is None:
        pytest.skip("g++ not available")
    return L


def _batch(seed, dtype, counts, integer=False):
    rng = np.random.default_rng(seed)
    imgs = [C.image(rng, h, w, dtype) for h, w in SHAPES]
    quads = []
    for n, (h, w) in enumerate(SHAPES):
        q, _ = C.quads(seed * 10 + n, counts[n], h, w)
        quads.append(np.round(q).astype(np.int32) if integer else q)
    return imgs, quads


def _expected(lib, imgs, quads, size, mode):
    rows = []
    for img, qs in zip(imgs, quads):
        for q in qs:
            rows.append(C.host_crop(lib, img, q.astype(np.float32), size, mode).transpose(2, 0, 1))
    return np.stack(rows) if rows else np.zeros((0, 3) + tuple(size), np.float32)


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("mode", ["resize", "pad"])
def test_packed_float_quads_match_harness(lib, dtype, mode):
    imgs, quads = _batch(3, dtype, [25, 0, 30])
    dev = torch.device("cuda")
    out = text_crop.crop_quads([torch.from_numpy(i).to(dev) for i in imgs], [torch.from_numpy(q).to(dev) for q in quads],
                               image_size=(32, 100), mode=mode)
    want = _expected(lib, imgs, quads, (32, 100), mode)
    assert int(out["total"][0]) == 55
    np.testing.assert_array_equal(out["image"].cpu().numpy(), want)
    owner = out["owner"].cpu().numpy()
    assert owner[:25, 0].tolist() == [0] * 25 and owner[25:, 0].tolist() == [2] * 30
    assert owner[25:, 1].tolist() == list(range(30))
    st = out["status"].cpu().numpy()
    assert not (st & 15).any() and st[0] & 16        # the degenerate kinds take the source's size


def test_int_boxes_with_counts_and_overflow(lib):
    imgs, quads = _batch(4, np.uint8, [12, 7, 9], integer=True)
    K = 12
    boxes = np.zeros((3, K, 4, 2), np.int32)
    for n, q in enumerate(quads):
        boxes[n, :len(q)] = q
    dev = torch.device("cuda")
    buf, offs, shapes = db_batch.pack_images([torch.from_numpy(i).to(dev) for i in imgs])
    counts = torch.tensor([len(q) for q in quads], dtype=torch.int32, device=dev)
    out = text_crop.crop_quads_packed(buf, offs, shapes, torch.from_numpy(boxes).to(dev), counts, (64, 256))
    want = _expected(lib, imgs, quads, (64, 256), "resize")
    np.testing.assert_array_equal(out["image"][:28].cpu().numpy(), want)
    assert (out["owner"][28:] == -1).all()
    small = text_crop.crop_quads_packed(buf, offs, shapes, torch.from_numpy(boxes).to(dev), counts, (64, 256), capacity=15)
    assert int(small["total"][0]) == 28
    np.testing.assert_array_equal(small["image"].cpu().numpy(), want[:15])
    st = small["status"].cpu().numpy()
    assert not st[0] & 8 and st[1] & 8 and st[2] & 8


def test_graph_replay_with_new_inputs(lib):
    dev = torch.device("cuda")
    imgs, quads = _batch(5, np.uint8, [10, 4, 6])
    imgs2, quads2 = _batch(6, np.uint8, [10, 4, 6])
    buf, offs, shapes = db_batch.pack_images([torch.from_numpy(i).to(dev) for i in imgs])
    q = torch.from_numpy(np.concatenate(quads)).to(dev)
    o = torch.tensor([0, 10, 14, 20], dtype=torch.int32, device=dev)
    text_crop.crop_quads_packed(buf, offs, shapes, q, o, (32, 100))
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = text_crop.crop_quads_packed(buf, offs, shapes, q, o, (32, 100))
    buf2, _, _ = db_batch.pack_images([torch.from_numpy(i).to(dev) for i in imgs2])
    buf.copy_(buf2)
    q.copy_(torch.from_numpy(np.concatenate(quads2)).to(dev))
    g.replay()
    eager = text_crop.crop_quads_packed(buf, offs, shapes, q, o, (32, 100))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out["image"].cpu().numpy(), eager["image"].cpu().numpy())
    np.testing.assert_array_equal(out["image"].cpu().numpy(), _expected(lib, imgs2, quads2, (32, 100), "resize"))


def test_image_cropper_returns_hwc(lib):
    rng = np.random.default_rng(9)
    img = C.image(rng, 120, 200, np.uint8)
    q, _ = C.quads(9, 1, 120, 200)
    got = text_crop.ImageCropper((32, 100)).crop(torch.from_numpy(img).cuda(), torch.from_numpy(q[0]).cuda())
    np.testing.assert_array_equal(got.cpu().numpy(), C.host_crop(lib, img, q[0], (32, 100)))


def test_refusals():
    L = _lib.lib()
    assert L.mr_text_crop_workspace_bytes(0, 10) == 0 and L.mr_text_crop_workspace_bytes(2, 70000) == 0
    nb = int(L.mr_text_crop_workspace_bytes(2, 4))
    d = torch.empty(4096, dtype=torch.uint8, device="cuda")
    p = d.data_ptr()
    args = lambda **k: dict(dict(image_dtype=0, N=2, quad_dtype=0, K=2, rows=4, cap=4, mode=0, oh=32, ow=100, ws=nb), **k)  # noqa
    for bad in (dict(N=0), dict(image_dtype=2), dict(quad_dtype=3), dict(mode=2), dict(oh=0), dict(ow=0), dict(ws=nb - 1),
                dict(K=-1), dict(rows=5)):
        a = args(**bad)
        rc = L.mr_text_crop(p, a["image_dtype"], 100, p, p, a["N"], p, a["quad_dtype"], a["rows"], a["K"], p, a["cap"], a["mode"],
                            a["oh"], a["ow"], 0.0, 0.0, 0.0, p, a["ws"], p, p, p, p, None)
        assert rc == 4, bad
    with pytest.raises(ValueError):
        text_crop.ImageCropper(mode="keep_ratio")
    with pytest.raises(NotImplementedError):
        text_crop.crop_quads_packed(torch.zeros(3, dtype=torch.uint8), None, None, None, None)


def _maps_and_boxes(seed, dev, n=3, map_hw=(96, 160), img_hw=(192, 320), per=5):
    """binary maps drawn from known quads, and boxes_from_maps' int32 boxes rescaled to the image size"""
    import cv2
    from megreader_b200 import db_boxes
    rng = np.random.default_rng(seed)
    maps = np.zeros((n, 1) + map_hw, np.float32)
    centres = [(30 + 50 * j, 25 + 45 * i) for i in range(2) for j in range(3)][:per]
    for k in range(n):
        for cx, cy in centres:             # separate rotated text-like boxes, 36 x 10 map pixels
            a = rng.uniform(-0.3, 0.3)
            r = np.array([[np.cos(a), np.sin(a)], [-np.sin(a), np.cos(a)]])
            q = np.array([(-18, -5), (18, -5), (18, 5), (-18, 5)]) @ r + (cx + rng.uniform(-3, 3), cy + rng.uniform(-3, 3))
            cv2.fillPoly(maps[k, 0], [np.round(q).astype(np.int32)], 0.9)
    sizes = torch.tensor([img_hw] * n, dtype=torch.int32, device=dev)
    boxes, _, count = db_boxes.boxes_from_maps(torch.from_numpy(maps).to(dev), max_candidates=20, dest_sizes=sizes)
    return torch.from_numpy(maps).to(dev), sizes, boxes, count


def test_boxes_from_maps_input(lib):
    dev = torch.device("cuda")
    maps, sizes, boxes, count = _maps_and_boxes(7, dev)
    rng = np.random.default_rng(7)
    imgs = [C.image(rng, 192, 320, np.uint8) for _ in range(3)]
    buf, offs, shapes = db_batch.pack_images([torch.from_numpy(i).to(dev) for i in imgs])
    out = text_crop.crop_quads_packed(buf, offs, shapes, boxes, count, (32, 128))
    cnt = count.cpu().numpy()
    assert cnt.sum() > 6 and int(out["total"][0]) == cnt.sum()
    b = boxes.cpu().numpy()
    want = _expected(lib, imgs, [b[n, :cnt[n]] for n in range(3)], (32, 128), "resize")
    np.testing.assert_array_equal(out["image"][:cnt.sum()].cpu().numpy(), want)
    empty = text_crop.crop_quads_packed(buf, offs, shapes, boxes[:, :0], torch.zeros(3, dtype=torch.int32, device=dev), (32, 128))
    assert empty["image"].shape[0] == 0 and int(empty["total"][0]) == 0


def test_detection_to_strings_chain_in_one_graph(lib):
    """boxes_from_maps -> crop_quads_packed -> engine CRNN eval -> ctc_greedy_decode captured as one CUDA graph: a replay with
    new maps and images equals the eager chain, and its crops equal the harness on the boxes it found"""
    import bench
    from megreader_b200 import db_boxes, decode
    dev = torch.device("cuda")
    torch.manual_seed(0)
    net = bench.build_model(dev).eval()
    rng = np.random.default_rng(11)
    inputs = []
    for s in (21, 22):
        maps, sizes, _, _ = _maps_and_boxes(s, dev)
        imgs = [C.image(rng, 192, 320, np.uint8) for _ in range(3)]
        inputs.append((maps, imgs))
    buf, offs, shapes = db_batch.pack_images([torch.from_numpy(i).to(dev) for i in inputs[0][1]])
    static_maps = inputs[0][0].clone()

    def chain():
        boxes, _, count = db_boxes.boxes_from_maps(static_maps, max_candidates=20, dest_sizes=sizes)
        crops = text_crop.crop_quads_packed(buf, offs, shapes, boxes, count, (32, 128))
        labels = decode.ctc_greedy_decode(net.decoder(net.backbone(crops["image"]), train=False))
        return boxes, count, crops, labels

    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            chain()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            res = chain()
        maps2, imgs2 = inputs[1]
        static_maps.copy_(maps2)
        buf.copy_(db_batch.pack_images([torch.from_numpy(i).to(dev) for i in imgs2])[0])
        g.replay()
        eager = chain()
        torch.cuda.synchronize()
    total = int(res[2]["total"][0])
    assert total == int(eager[2]["total"][0]) and total > 6
    np.testing.assert_array_equal(res[2]["image"][:total].cpu().numpy(), eager[2]["image"][:total].cpu().numpy())
    lab_g, lab_e = (res[3][0], eager[3][0]) if isinstance(res[3], tuple) else (res[3], eager[3])
    assert torch.equal(lab_g[:total], lab_e[:total])
    cnt, b = res[1].cpu().numpy(), res[0].cpu().numpy()
    want = _expected(lib, imgs2, [b[n, :cnt[n]] for n in range(3)], (32, 128), "resize")
    np.testing.assert_array_equal(res[2]["image"][:total].cpu().numpy(), want)


def test_golden_on_device(lib):
    """The device's crops of the golden's cases equal the reference's sampled values (cv2 unoptimised) wherever the rectangle
    and matrix are cv2's, and the harness everywhere"""
    import os
    from oracle import text_crop_port as port
    from oracle.make_text_crop_golden import CASES, case_inputs
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_crop_ref.npz"))
    dev = torch.device("cuda")
    for i, (name, dtype, mode, size) in enumerate(CASES):
        img, q, _ = case_inputs(i, dtype)
        out = text_crop.crop_quads([torch.from_numpy(img).to(dev)], [torch.from_numpy(q).to(dev)], image_size=size, mode=mode)
        got = out["image"].permute(0, 2, 3, 1).cpu().numpy()
        geo = C.host_setup(lib, q, *img.shape[:2], mode, size)
        idx = g[name + "/index"]
        compared = 0
        for k in range(len(q)):
            np.testing.assert_array_equal(got[k], C.host_crop(lib, img, q[k], size, mode), err_msg="%s %d" % (name, k))
            if np.array_equal(port.min_area_rect(q[k]), geo["box"][k]) and geo["P"][k].reshape(-1)[:8].any():
                np.testing.assert_array_equal(got[k].reshape(-1)[idx], g[name + "/plain"][k], err_msg="%s %d" % (name, k))
                np.testing.assert_array_equal(got[k].astype(np.float64).sum((0, 1)), g[name + "/sums"][k])
                compared += 1
        assert compared >= len(q) // 2, name
