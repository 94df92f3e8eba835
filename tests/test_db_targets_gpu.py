"""GPU: megreader_b200.db_targets (csrc/db_targets.cu) bit for bit against the golden made by the reference's own
MakeSegDetectionData / MakeBorderMap classes (tests/golden/db_targets_ref.npz, oracle/make_db_targets_golden.py) and against
the live oracle (oracle/db_targets_port.py): the four maps, the validated polygons, the ignore tags and the per-polygon
status, for float32 and float64 polygons; a captured graph replayed with new polygons; bad inputs refused without a fault;
and resize_normalize at an image's own size against NormalizeImage."""
import os

import numpy as np
import pytest
import torch

from oracle import db_targets_port as port
from tests.db_targets_cases import batch

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "db_targets_ref.npz")
MAPS = ("gt", "mask", "thresh_map", "thresh_mask")


def run(images, H, W, dtype):
    from megreader_b200 import db_targets
    polys = [torch.as_tensor(np.asarray(p, dtype).reshape(-1, 4, 2), device="cuda") for p, _ in images]
    tags = [torch.as_tensor(np.asarray(t, bool).reshape(-1), device="cuda") for _, t in images]
    out = db_targets.make_targets(polys, tags, (H, W))
    torch.cuda.synchronize()
    return out


def assert_bits(got, want, what):
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    bad = got.view(np.uint8) != want.view(np.uint8)
    assert not bad.any(), (what, np.argwhere(bad.reshape(got.shape[0], -1) if got.ndim else bad)[:5])


def check_against_oracle(images, H, W, dtype):
    out = run(images, H, W, dtype)
    for n, (p, t) in enumerate(images):
        want = port.make_targets(np.asarray(p, dtype).reshape(-1, 4, 2).copy(), t, (H, W))
        assert_bits(out["gt"][n].cpu().numpy(), want["gt"], "gt %d" % n)
        for k in ("mask", "thresh_map", "thresh_mask"):
            assert_bits(out[k][n].cpu().numpy(), want[k], "%s %d" % (k, n))
        assert_bits(out["polygons"][n].cpu().numpy(), want["polygons"], "polygons %d" % n)
        assert_bits(out["ignore_tags"][n].cpu().numpy(), want["ignore_tags"], "ignore_tags %d" % n)
        assert_bits(out["status"][n].cpu().numpy(), want["status"], "status %d" % n)
    return out


def decode_values(planes):
    """inverse of oracle/make_db_targets_golden.encode_values: byte planes of bit-pattern differences -> float32 values"""
    d = np.ascontiguousarray(planes.T).view(np.uint32).reshape(-1)
    return np.cumsum(d, dtype=np.uint32).view(np.float32)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("case", ["b640", "f32", "wide", "odd"])
def test_golden(golden, case):
    N, H, W = (int(v) for v in golden[case + "/size"])
    counts = golden[case + "/counts"]
    ends = np.concatenate([[0], np.cumsum(counts)])
    pin, tin = golden[case + "/polygons_in"], golden[case + "/tags_in"]
    images = [(pin[ends[i]:ends[i + 1]], tin[ends[i]:ends[i + 1]]) for i in range(N)]
    out = run(images, H, W, pin.dtype)
    for k in ("gt", "mask", "thresh_mask"):
        want = np.unpackbits(golden[case + "/" + k])[:N * H * W].reshape(N, H, W).astype(np.float32)
        assert_bits(out[k].reshape(N, H, W).cpu().numpy(), want, k)
    tm = np.full((N, H, W), np.float32(0.3))
    at = np.unpackbits(golden[case + "/thresh_map_at"])[:N * H * W].reshape(N, H, W).astype(bool)
    tm[at] = decode_values(golden[case + "/thresh_map_planes"])
    assert_bits(out["thresh_map"].cpu().numpy(), tm, "thresh_map")
    assert_bits(torch.cat(out["polygons"]).cpu().numpy(), golden[case + "/polygons"], "polygons")
    assert_bits(torch.cat(out["ignore_tags"]).cpu().numpy(), golden[case + "/ignore_tags"], "ignore_tags")
    assert_bits(torch.cat(out["status"]).cpu().numpy(), golden[case + "/status"], "status")


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_batch16_640(dtype):
    images = batch(10, 16, 640, 640, 0, 60, dtype, odd=0.3)
    out = check_against_oracle(images, 640, 640, dtype)
    st = torch.cat(out["status"]).cpu().numpy()
    assert (st & port.SMALL_TEXT).any() and (st & port.TINY_AREA).any()


def test_wide_batch():
    check_against_oracle(batch(11, 4, 576, 1024, 5, 40, np.float64, odd=0.4), 576, 1024, np.float64)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_odd_quads(dtype):
    """sub-8 px text, |area| < 1, duplicate corners, concave and bow-tie quads, slivers, border-clipped quads with NaN pixels"""
    images = batch(12, 6, 200, 300, 10, 30, dtype, odd=1.0)
    check_against_oracle(images, 200, 300, dtype)


def test_one_image_no_polygons_and_all_ignored():
    out = check_against_oracle([(np.zeros((0, 4, 2)), np.zeros(0, bool))], 64, 96, np.float64)
    assert out["mask"].min().item() == 1 and out["gt"].max().item() == 0
    assert (out["thresh_map"] == np.float32(0.3)).all()
    polys, _ = batch(13, 1, 64, 96, 8, 8, np.float64, odd=0.0)[0]
    out = check_against_oracle([(polys, np.ones(8, bool))], 64, 96, np.float64)
    assert out["gt"].max().item() == 0 and out["thresh_mask"].max().item() == 0


def test_graph_replay_with_new_polygons():
    from megreader_b200 import db_targets
    H, W, cap = 320, 320, 64
    first = batch(14, 3, H, W, 5, 20, np.float64)
    second = batch(15, 3, H, W, 5, 20, np.float64)

    def packed(images):
        return db_targets.pack([torch.as_tensor(p, device="cuda") for p, _ in images],
                               [torch.as_tensor(t, device="cuda") for _, t in images], cap)

    polys, tags, offsets = packed(first)
    db_targets.make_targets_packed(polys, tags, offsets, (H, W))        # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = db_targets.make_targets_packed(polys, tags, offsets, (H, W))
    p2, t2, o2 = packed(second)
    polys.copy_(p2)
    tags.copy_(t2)
    offsets.copy_(o2)
    g.replay()
    torch.cuda.synchronize()
    eager = db_targets.make_targets_packed(p2, t2, o2, (H, W))
    torch.cuda.synchronize()
    for k in MAPS + ("polygons", "ignore_tags", "status"):
        assert torch.equal(out[k], eager[k]), k


def test_bad_inputs_refused():
    from megreader_b200 import _lib, db_targets
    p = torch.zeros((2, 4, 2), dtype=torch.float64)
    t = torch.zeros(2, dtype=torch.bool)
    with pytest.raises(NotImplementedError):
        db_targets.make_targets([p], [t], (32, 32))
    with pytest.raises(RuntimeError):
        db_targets.make_targets([p.cuda().float().reshape(2, 8)], [t.cuda()], (32, 32))
    with pytest.raises(RuntimeError):
        db_targets.make_targets([p.cuda().int()], [t.cuda()], (32, 32))
    with pytest.raises(RuntimeError):
        db_targets.make_targets([p.cuda()], [t.cuda()], (0, 32))
    L = _lib.lib()
    assert L.mr_db_targets_workspace_bytes(1, 1 << 15, 1 << 15, 4) == 0
    polys, tags, offsets = db_targets.pack([p.cuda()], [t.cuda()])
    nbytes = int(L.mr_db_targets_workspace_bytes(1, 32, 32, 2))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    maps = torch.empty((4, 32, 32), device="cuda")
    po, io, st = torch.empty_like(polys), torch.empty_like(tags), torch.empty(2, dtype=torch.int32, device="cuda")
    args = lambda dtype, nb: (polys.data_ptr(), dtype, tags.data_ptr(), offsets.data_ptr(), 1, 32, 32, 2, 0.84, 8.0,  # noqa: E731
                              0.4, 0.3, ws.data_ptr(), nb, maps[0].data_ptr(), maps[1].data_ptr(), maps[2].data_ptr(),
                              maps[3].data_ptr(), po.data_ptr(), io.data_ptr(), st.data_ptr(), None)
    assert L.mr_db_targets(*args(2, nbytes)) != 0                      # unknown dtype
    assert L.mr_db_targets(*args(1, nbytes - 1)) != 0                  # workspace too small
    assert L.mr_db_targets(*args(1, nbytes)) == 0
    torch.cuda.synchronize()


def test_resize_normalize_equals_normalize_image():
    """NormalizeImage (data/processes/normalize_image.py): image -= RGB_MEAN; image /= 255.; CHW -- against
    input_pipeline.resize_normalize at the image's own size"""
    from megreader_b200 import input_pipeline
    rng = np.random.default_rng(16)
    mean = np.array([122.67891434, 116.66876762, 104.00698793])
    for H, W in ((640, 640), (37, 91)):
        img = (rng.random((H, W, 3)) * 255).astype(np.float32)
        want = img.copy()
        want -= mean
        want /= 255.
        want = np.ascontiguousarray(want.transpose(2, 0, 1))
        got = input_pipeline.resize_normalize([img], (H, W)).cpu().numpy()[0]
        assert_bits(got, want, "normalize %dx%d" % (H, W))
