"""CPU: the PRODUCT's DB input-batch routines (megreader_b200/csrc/db_batch_core.cuh -- the code the CUDA kernels of
csrc/db_batch.cu run) compiled for the host by tests/host_harness/db_batch_core_host.cpp, checked against
  * the golden (tests/golden/db_batch_ref.npz, from the reference's own RandomCropData): crop rectangles, scales, kept quads
    and tags bit for bit, and the stored pixel samples;
  * the oracle (oracle/db_batch_port.py) on a few thousand seeded polygon sets, including empty, all-ignored and
    second-round cases, and the reference's RandomCropData live where the reference tree is present;
  * cv2.warpAffine and cv2.resize (INTER_CUBIC, INTER_LINEAR) on seeded float32 images, with cv2's optimisations off and on;
  * the keypoint convention: a dot drawn at a quad corner lands within one pixel of the transformed corner."""
import os

import numpy as np
import pytest

from oracle import db_batch_port as port
from tests import db_batch_cases as C

cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "db_batch_ref.npz")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    L = C.build_harness(tmp_path_factory.mktemp("harness"))
    if L is None:
        pytest.skip("g++ not available")
    return L


@pytest.fixture
def optimized():
    was = cv2.useOptimized()
    yield
    cv2.setUseOptimized(was)


def test_golden_geometry_and_pixels(lib):
    g = np.load(GOLDEN)
    for i, (name, *_) in enumerate(C.CASES):
        c = C.case(name)
        h, w = c["image"].shape[:2]
        geo = C.host_geometry(lib, c["mode"], h, w, c["polys"], c["tags"], c["draws"])
        np.testing.assert_array_equal(g[name + "/draws"], c["draws"])
        assert list(geo["crop"]) == g[name + "/crop"].tolist(), name
        assert geo["scale"] == float(g[name + "/scale"]), name
        np.testing.assert_array_equal(geo["polygons"], g[name + "/polygons"], err_msg=name)
        np.testing.assert_array_equal(geo["ignore_tags"], g[name + "/ignore_tags"], err_msg=name)
        img = C.host_output(lib, c["mode"], c["image"], geo, c["draws"])
        np.testing.assert_array_equal(img.reshape(-1)[C.pixel_sample(i, img.shape)], g[name + "/host_pixels"], err_msg=name)


def test_golden_covers_the_crop_cases():
    g = np.load(GOLDEN)
    rounds = {name: int(g[name + "/round"]) for name, _, mode, *_ in C.CASES if mode == "train"}
    assert rounds["crop640"] == 0 and rounds["second_round"] == 1 and rounds["no_care"] == 2
    assert g["crop640/crop"].tolist()[2:] == [640, 640]
    assert len(g["dropped/polygons"]) < len(C.case("dropped")["polys"])
    assert any(g[name + "/ignore_tags"].any() for name, _, mode, *_ in C.CASES if mode == "train")
    assert C.case("no_care")["tags"].all()
    c = C.case("negative")
    _, aug, _ = port.augment(c["image"].astype(np.float32), c["polys"], c["draws"])
    assert (np.round(aug) < 0).any()
    assert C.case("scale3_max")["image"].shape[:2] == (C.MAX_H, C.MAX_W) and C.case("scale3_max")["draws"][2] == 1.0


def test_crop_rule_against_oracle(lib):
    n = 0
    for h, w, q, tags, u in C.polygon_sets(17, 3000):
        geo = C.host_geometry(lib, "train", h, w, q, tags, u)
        img = np.zeros((h, w, 3), np.float32)
        _, aug, (flip, deg, hs, ws) = port.augment(img, q, u)
        np.testing.assert_array_equal(geo["augmented"], aug)
        assert (geo["hs"], geo["ws"], geo["flip"]) == (hs, ws, flip)
        care = [p for p, t in zip(aug, tags) if not t]
        cx, cy, cw, ch, _ = port.crop_area(hs, ws, care, port.Picks(u, 10), 640, 10, 0.1)
        assert geo["crop"] == (cx, cy, cw, ch)
        scale = min(640 / cw, 640 / ch)
        assert geo["scale"] == scale
        kept = [(p - (cx, cy)) * scale for p in aug]
        keep = [not port.outside(p, 0, 0, int(cw * scale), int(ch * scale)) for p in kept]
        np.testing.assert_array_equal(geo["polygons"], np.array([p for p, k in zip(kept, keep) if k]).reshape(-1, 4, 2))
        n += 1
    assert n == 3000


def test_crop_rule_against_reference(lib):
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("reference tree not present")
    from oracle import make_db_batch_golden as mk
    rc, icdar, norm = mk.reference_processes()
    for h, w, q, tags, u in list(C.polygon_sets(23, 300)):
        geo = C.host_geometry(lib, "train", h, w, q, tags, u)
        _, rect, _ = mk.reference_train(rc, icdar, norm, np.zeros((h, w, 3), np.uint8), q, tags, u)
        assert geo["crop"] == rect


def _images(seed, count):
    rng = np.random.default_rng(seed)
    for t in range(count):
        h, w = int(rng.integers(3, 200)), int(rng.integers(3, 200))
        img = (rng.random((h, w, 3)) * 255).astype(np.float32)
        yield rng, t, h, w, img


def _warp(lib, img, flip, deg):
    import ctypes
    out = np.zeros_like(img)
    lib.host_warp(C._p(img), img.shape[0], img.shape[1], int(flip), ctypes.c_double(deg), C._p(out))
    return out


def _resize(lib, fn, img, dh, dw):
    out = np.zeros((dh, dw, 3), np.float32)
    getattr(lib, fn)(C._p(img), img.shape[0], img.shape[1], dh, dw, C._p(out))
    return out


@pytest.mark.parametrize("opt", [False, True])
def test_warp_equals_cv2(lib, optimized, opt):
    cv2.setUseOptimized(opt)
    for rng, t, h, w, img in _images(3, 40):
        deg = float(rng.uniform(-10, 10))
        src = np.ascontiguousarray(img[:, ::-1]) if t % 2 else img
        ref = cv2.warpAffine(src, port.rotation_matrix(deg, w, h), (w, h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT,
                             borderValue=0)
        np.testing.assert_array_equal(_warp(lib, img, t % 2, deg), ref)


# Largest |harness - cv2| on 0..255 float32 images over these seeds (cv2 4.13, x86-64); recorded in DESIGN §7
BOUNDS = {("cubic", False): 1e-4, ("cubic", True): 6e-3, ("linear", False): 0.0, ("linear", True): 4e-3}


@pytest.mark.parametrize("kind", ["cubic", "linear"])
@pytest.mark.parametrize("opt", [False, True])
def test_resize_against_cv2(lib, optimized, kind, opt):
    cv2.setUseOptimized(opt)
    worst, differ, total = 0.0, 0, 0
    for rng, t, h, w, img in _images(5, 40):
        s = float(rng.uniform(0.5, 3.0))
        dh, dw = max(1, round(h * s)), max(1, round(w * s))
        ref = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_CUBIC if kind == "cubic" else cv2.INTER_LINEAR)
        got = _resize(lib, "host_" + kind, img, dh, dw)
        worst = max(worst, float(np.abs(got - ref).max()))
        differ += int((got != ref).sum())
        total += got.size
    assert worst <= BOUNDS[(kind, opt)], worst
    if kind == "cubic" and not opt:            # only cv2's scalar row tails add in the other order
        assert differ < 0.01 * total


def test_validation_resize_equals_cv2_cubic(lib):
    c = C.case("validate")
    h, w = c["image"].shape[:2]
    geo = C.host_geometry(lib, "validate", h, w, c["polys"], c["tags"], c["draws"])
    got = C.host_output(lib, "validate", c["image"], geo, c["draws"])
    ref = port.validate_sample(c["image"], c["polys"], c["tags"])
    assert np.abs(got - ref["image"]).max() <= 2.5e-5
    np.testing.assert_array_equal(geo["polygons"], ref["polygons"])


def test_keypoints_follow_the_pixels(lib):
    """A one-pixel dot at each quad corner, pushed through the harness's warp and cubic resize, peaks within one pixel of the
    corner the keypoint rules give (pins the flip's w - x, the rotation centre and the resize's (x / w) * new_w)."""
    rng = np.random.default_rng(9)
    for t in range(60):
        h, w = int(rng.integers(40, 160)), int(rng.integers(40, 160))
        x, y = int(rng.integers(5, w - 5)), int(rng.integers(5, h - 5))
        img = np.zeros((h, w, 3), np.float32)
        img[y, x] = 255.
        u = rng.random(83).astype(np.float32)
        u[0] = 0.2 if t % 2 else 0.8
        geo = C.host_geometry(lib, "train", h, w, np.array([[[x + .5, y + .5]] * 4]), np.ones(1, np.uint8), u)
        warped = _warp(lib, img, geo["flip"], port.params(u)[1])
        out = _resize(lib, "host_cubic", warped, geo["hs"], geo["ws"])
        py, px = np.unravel_index(np.argmax(out[..., 0]), out.shape[:2])
        kx, ky = geo["augmented"][0, 0, 0] - 0.5, geo["augmented"][0, 0, 1] - 0.5     # keypoint -> pixel index (centres at +0.5)
        tol = 1.0 + 0.5 * geo["ws"] / w
        assert abs(px - kx) <= tol and abs(py - ky) <= tol, (t, px, py, kx, ky)
