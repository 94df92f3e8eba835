"""GPU: the DB input batch (megreader_b200.db_batch, csrc/db_batch.cu) against tests/golden/db_batch_ref.npz, built with
the reference's own RandomCropData / MakeICDARData / NormalizeImage after the restated augmentation:
  * crop rectangles, scales, kept quads, tags and offsets exactly, for all training cases in one ragged batch (uint8 and
    float32 pixels) and for the validation case;
  * the normalised pixels bit-equal to the host harness's values and within the CPU-measured bound of the cv2 chain;
  * train_batch_packed + make_targets_packed captured in one CUDA graph and replayed with new images and draws;
  * validate_batch through SegDetectorRepresenter and QuadMeasurer unchanged;
  * the per-image status of an oversized input, bad offsets and refused calls."""
import os

import numpy as np
import pytest
import torch

from megreader_b200 import db_batch, db_boxes, db_measure, db_targets
from tests import db_batch_cases as C

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "db_batch_ref.npz")
CV2_BOUND = 2.5e-5          # normalised units (about 0.0064 on 0..255): cv2's vectorised cubic / linear resize, DESIGN §7
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _inputs(names, img_dtype, poly_dtype):
    cases = [C.case(n) for n in names]
    imgs = [torch.from_numpy(c["image"]).to(DEV).to(img_dtype) for c in cases]
    polys = [torch.from_numpy(c["polys"]).to(DEV).to(poly_dtype) for c in cases]
    tags = [torch.from_numpy(c["tags"]).to(DEV) for c in cases]
    return cases, imgs, polys, tags


def _check(out, names, golden):
    torch.cuda.synchronize()
    assert out["status"].tolist() == [0] * len(names)
    offs = out["offsets"].cpu().numpy()
    polys, tags = out["polygons"].cpu().numpy(), out["ignore_tags"].cpu().numpy()
    img = out["image"].cpu().numpy()
    for n, name in enumerate(names):
        assert out["crop"][n].tolist() == golden[name + "/crop"].tolist(), name
        assert float(out["scale"][n]) == float(golden[name + "/scale"]), name
        h, w = C.case(name)["image"].shape[:2]
        assert out["shape"][n].tolist() == [h, w]
        np.testing.assert_array_equal(polys[offs[n]:offs[n + 1]], golden[name + "/polygons"], err_msg=name)
        np.testing.assert_array_equal(tags[offs[n]:offs[n + 1]], golden[name + "/ignore_tags"], err_msg=name)
        idx = C.pixel_sample(list(g[0] for g in C.CASES).index(name), img[n].shape)
        np.testing.assert_array_equal(img[n].reshape(-1)[idx], golden[name + "/host_pixels"], err_msg=name)
        np.testing.assert_allclose(img[n].astype(np.float64).sum((1, 2)), golden[name + "/host_sums"], rtol=1e-6, atol=1e-3)
        assert np.abs(img[n].reshape(-1)[idx] - golden[name + "/ref_pixels"]).max() <= CV2_BOUND, name
    assert (polys[offs[-1]:] == 0).all() and (tags[offs[-1]:] == 0).all()


TRAIN = [c[0] for c in C.CASES if c[2] == "train"]


@pytest.mark.parametrize("img_dtype", [torch.uint8, torch.float32])
def test_train_golden(golden, img_dtype):
    cases, imgs, polys, tags = _inputs(TRAIN, img_dtype, torch.float64)
    buf, ioff, shapes = db_batch.pack_images(imgs)
    P, T, O = db_targets.pack(polys, tags, capacity=sum(len(c["polys"]) for c in cases) + 5)
    u = torch.from_numpy(np.stack([c["draws"] for c in cases])).to(DEV)
    out = db_batch.train_batch_packed(buf, ioff, shapes, C.MAX_H, C.MAX_W, P, T, O, u)
    _check(out, TRAIN, golden)


def test_validate_golden(golden):
    cases, imgs, polys, tags = _inputs(["validate"], torch.uint8, torch.float64)
    buf, ioff, shapes = db_batch.pack_images(imgs)
    P, T, O = db_targets.pack(polys, tags)
    out = db_batch.validate_batch_packed(buf, ioff, shapes, C.MAX_H, C.MAX_W, P, T, O)
    _check(out, ["validate"], golden)


def test_graph_replay():
    names = TRAIN[:4]
    cases, imgs, polys, tags = _inputs(names, torch.uint8, torch.float64)
    buf, ioff, shapes = db_batch.pack_images(imgs)
    P, T, O = db_targets.pack(polys, tags, capacity=64)
    u = torch.rand((len(names), db_batch.draws_per_image()), device=DEV)

    def step():
        out = db_batch.train_batch_packed(buf, ioff, shapes, C.MAX_H, C.MAX_W, P, T, O, u)
        t = db_targets.make_targets_packed(out["polygons"], out["ignore_tags"], out["offsets"], (640, 640))
        return out, t
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out_g, t_g = step()
    gen = torch.Generator(device=DEV).manual_seed(11)
    for _ in range(3):
        buf.copy_(torch.randint(0, 256, buf.shape, generator=gen, device=DEV, dtype=torch.uint8))
        u.copy_(torch.rand(u.shape, generator=gen, device=DEV))
        g.replay()
        out_e, t_e = step()
        torch.cuda.synchronize()
        for k in ("image", "polygons", "ignore_tags", "offsets", "crop", "scale", "status"):
            assert torch.equal(out_g[k], out_e[k]), k
        for k in ("gt", "mask", "thresh_map", "thresh_mask"):
            assert torch.equal(t_g[k], t_e[k]), k


def test_validate_batch_through_boxes_and_measure():
    rng = np.random.default_rng(5)
    imgs, polys, tags = [], [], []
    for h, w in ((410, 530), (576, 1024), (300, 700), (700, 500)):
        imgs.append(torch.from_numpy(C.image(rng, h, w)).to(DEV))
        polys.append(torch.from_numpy(C.quads(rng, h, w, 6)).to(DEV))
        tags.append(torch.from_numpy((rng.random(6) < 0.2).astype(np.uint8)).to(DEV))
    batch = db_batch.validate_batch(imgs, polys, tags)
    assert batch["image"].shape == (4, 3, 576, 1024) and batch["gt"].shape == (4, 1, 576, 1024)
    assert batch["shape"].tolist() == [[410, 530], [576, 1024], [300, 700], [700, 500]]
    pred = dict(binary=batch["gt"], thresh=batch["thresh_map"], thresh_binary=batch["gt"])
    boxes, _ = db_boxes.SegDetectorRepresenter().represent(batch, pred)
    res = db_measure.QuadMeasurer().measure(batch, (boxes, pred))
    assert len(res) == 4 and sum(r["detMatched"] for r in res) > 0


def test_status_and_refusals():
    cases, imgs, polys, tags = _inputs(["crop640", "flip_small"], torch.uint8, torch.float64)
    buf, ioff, shapes = db_batch.pack_images(imgs)
    P, T, O = db_targets.pack(polys, tags)
    u = torch.rand((2, db_batch.draws_per_image()), device=DEV)
    out = db_batch.train_batch_packed(buf, ioff, shapes, 300, 300, P, T, O, u)     # image 0 (480 x 640) exceeds 300 x 300
    torch.cuda.synchronize()
    assert out["status"].tolist() == [db_batch.STATUS["bad_shape"], 0]
    assert out["offsets"].tolist()[:2] == [0, 0] and bool((out["image"][0] == out["image"][0, :, :1, :1]).all())
    bad = O.clone()
    bad[-1] = P.size(0) + 1                                                         # the offsets exceed the capacity
    out = db_batch.train_batch_packed(buf, ioff, shapes, C.MAX_H, C.MAX_W, P, T, bad, u)
    torch.cuda.synchronize()
    assert out["status"].tolist() == [db_batch.STATUS["bad_offsets"]] * 2 and out["offsets"].tolist() == [0, 0, 0]
    with pytest.raises(RuntimeError):
        db_batch.train_batch_packed(buf, ioff, shapes, C.MAX_H, C.MAX_W, P, T, O, u[:, :10])
    with pytest.raises(RuntimeError):
        db_batch.train_batch_packed(buf, ioff, shapes, C.MAX_H, C.MAX_W, P, T, O, u, scale=(0.5, 5.0))
    with pytest.raises(NotImplementedError):
        db_batch.pack_images([torch.zeros((4, 4, 3), dtype=torch.uint8)])
    with pytest.raises(RuntimeError):
        db_batch.train_batch_packed(buf, ioff, shapes[:1], C.MAX_H, C.MAX_W, P, T, O, u)


def test_train_batch_dict():
    cases, imgs, polys, tags = _inputs(TRAIN[:3], torch.uint8, torch.float64)
    out = db_batch.train_batch(imgs, polys, tags, generator=torch.Generator(device=DEV).manual_seed(3))
    assert sorted(out) == ["gt", "image", "mask", "thresh_map", "thresh_mask"]
    assert out["image"].shape == (3, 3, 640, 640) and out["gt"].shape == (3, 1, 640, 640)
    assert bool(torch.isfinite(out["image"]).all())
