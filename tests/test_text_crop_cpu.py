"""CPU: the PRODUCT's text-crop routines (megreader_b200/csrc/text_crop_core.cuh -- the code the CUDA kernels of csrc/text_crop.cu
run) compiled for the host by tests/host_harness/text_crop_core_host.cpp, checked against
  * the oracle (oracle/text_crop_port.py, cv2) on 10,000 seeded quads of every kind: the min-area rectangle, the float32 sides,
    the perspective matrix and its inverse, (int(w), int(h)) with the zero-side fallback and the turn, bit for bit except for
    the calipers tie class (DESIGN §7), which is counted and bounded;
  * cv2.warpPerspective on uint8 and float32 images, with cv2's optimisations on and off;
  * whole crops of both modes: bit for bit with cv2's optimisations off, within a measured bound with its defaults;
  * the reference's own ImageCropper, where the reference tree is present."""
import numpy as np
import pytest

from oracle import text_crop_port as port
from tests import text_crop_cases as C

cv2 = pytest.importorskip("cv2")

# The calipers class (DESIGN §7): per kind of quad, the largest share whose min-area rectangle differs from cv2.minAreaRect's
# (measured on the 10,000 seeded quads: thin 670, tall 687, diag45 634, int 29, rotated 13 and collinear 323 per 1,000), and
# how far its corners may then lie from cv2's (pixels, after matching the starting corner).  Collinear quads have a
# zero-width rectangle whose corners cv2 orders by another angle convention; their crops are checked below like all others.
TIE_SHARE = dict(thin=0.70, tall=0.72, diag45=0.66, int=0.035, rotated=0.02, collinear=0.35)
TIE_CORNER = dict(thin=0.05, tall=0.01, diag45=0.005, int=0.25, rotated=0.2)


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


def _singular(g, i):
    """The 8 x 8 system is singular (collinear or repeated corners): the product keeps LU's zero matrix, cv2 4.13 returns
    another solver's matrix (DESIGN §7)"""
    return not g["P"][i].reshape(-1)[:8].any()


def _same_geometry(g, i, q):
    box, w, h, P, size = port.crop_geometry(q)
    return np.array_equal(box, g["box"][i]) and not _singular(g, i), (box, w, h, P, size)


def test_geometry_against_oracle(lib):
    q, kinds = C.quads(11, 10000)
    g = C.host_setup(lib, q, 720, 1280)
    ties, zero, turned, singular = {}, 0, 0, 0
    for i in range(len(q)):
        same, (box, w, h, P, size) = _same_geometry(g, i, q[i])
        if _singular(g, i):
            singular += 1
            assert kinds[i] in ("point", "collinear"), (i, kinds[i])
            continue
        if not same:
            ties[kinds[i]] = ties.get(kinds[i], 0) + 1
            if kinds[i] != "collinear":
                dev = min(np.abs(np.roll(box.astype(np.float64), r, 0) - g["box"][i]).max() for r in range(4))
                assert dev <= TIE_CORNER[kinds[i]], (i, kinds[i], box, g["box"][i])
            continue
        assert (w, h) == tuple(g["sides"][i]), i
        np.testing.assert_array_equal(g["P"][i], P, err_msg="%d %s" % (i, kinds[i]))
        _, Minv = cv2.invert(P, flags=cv2.DECOMP_LU)
        np.testing.assert_array_equal(g["M"][i], Minv, err_msg="%d %s" % (i, kinds[i]))
        cw, ch = size if size[0] > 0 and size[1] > 0 else (1280, 720)
        assert tuple(g["size"][i][:2]) == (cw, ch), i
        assert bool(g["flags"][i] & 16) == (size[0] <= 0 or size[1] <= 0)
        assert g["turned"][i] == (ch > cw * 1.5)
        zero += bool(g["flags"][i] & 16)
        turned += bool(g["turned"][i])
    for kind, n in ties.items():
        assert n <= TIE_SHARE.get(kind, 0) * kinds.count(kind), ties
    assert zero > 100 and turned > 100 and singular <= 0.15 * len(q)


def test_perspective_singular_case(lib):
    """A quad of one point: LU finds the system singular and leaves the zero matrix (P[2, 2] = 1); the crop takes the source's
    size because both sides truncate to 0"""
    q = np.tile(np.float32([[10, 20]]), (4, 1))
    g = C.host_setup(lib, q, 50, 80)
    _, _, _, P, size = port.crop_geometry(q)
    assert g["P"][0][2, 2] == 1 and not g["P"][0].reshape(-1)[:8].any()
    assert tuple(g["size"][0][:2]) == (80, 50) and size == (0, 0) and g["flags"][0] & 16


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("opt", [False, True])
def test_warp_matches_cv2(lib, optimized, dtype, opt):
    cv2.setUseOptimized(opt)
    rng = np.random.default_rng(5)
    img = C.image(rng, 180, 260, dtype)
    q, kinds = C.quads(6, 300, 180, 260)
    g = C.host_setup(lib, q, 180, 260)
    for i in range(len(q)):
        P, size = g["P"][i], tuple(int(v) for v in g["size"][i][:2])
        ref = cv2.warpPerspective(img, P, size).astype(np.float32)
        np.testing.assert_array_equal(C.host_warp(lib, img, P, size), ref, err_msg="%d %s" % (i, kinds[i]))


def _crop_cases(lib, seed, dtype, count=120):
    rng = np.random.default_rng(seed)
    img = C.image(rng, 150, 230, dtype)
    q, kinds = C.quads(seed + 1, count, 150, 230)
    g = C.host_setup(lib, q, 150, 230)
    keep = [i for i in range(len(q)) if _same_geometry(g, i, q[i])[0]]
    return img, q, kinds, g, keep


def _cv2_crop(img, q, g, i, size, mode, same):
    """cv2's crop of quad i: the reference's own where the rectangle and matrix are cv2's, else cv2's warp, turn, resize and
    normalisation through the product's matrix and crop size"""
    if same:
        return port.crop(img, q, size, mode)
    return port.crop_with_matrix(img, g["P"][i], g["size"][i][:2], size, mode)


@pytest.mark.parametrize("mode", ["resize", "pad"])
@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_crops_bit_exact_unoptimised(lib, optimized, mode, dtype):
    cv2.setUseOptimized(False)
    img, q, kinds, g, keep = _crop_cases(lib, 21, dtype)
    assert len(keep) > 0.5 * len(q)
    assert g["turned"][keep].any() and (~g["turned"][keep]).any() and (g["flags"][keep] & 16).any()
    for size in ((32, 100), (64, 256)):
        for i in range(len(q)):
            ref = _cv2_crop(img, q[i], g, i, size, mode, i in keep)
            np.testing.assert_array_equal(C.host_crop(lib, img, q[i], size, mode), ref, err_msg="%d %s" % (i, kinds[i]))


# cv2's optimised INTER_LINEAR resize of float32 rounds its row blend differently from the plain one; measured largest
# difference of a normalised value on these cases
DEFAULT_BOUND = 1e-5


@pytest.mark.parametrize("mode", ["resize", "pad"])
def test_crops_with_cv2_defaults(lib, optimized, mode):
    cv2.setUseOptimized(True)
    worst = 0.0
    for dtype in (np.uint8, np.float32):
        img, q, kinds, g, keep = _crop_cases(lib, 31, dtype, 80)
        for i in range(len(q)):
            ref = _cv2_crop(img, q[i], g, i, (32, 100), mode, i in keep)
            worst = max(worst, float(np.abs(C.host_crop(lib, img, q[i], (32, 100), mode) - ref).max()))
    assert worst <= DEFAULT_BOUND, worst


def test_live_reference(lib, optimized):
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("reference tree not present")
    from oracle.make_text_crop_golden import reference_cropper
    cv2.setUseOptimized(False)
    cropper = reference_cropper((32, 100), "resize")
    img, q, kinds, g, keep = _crop_cases(lib, 41, np.uint8, 60)
    for i in keep:
        ref = cropper.crop(img, q[i])
        np.testing.assert_array_equal(port.crop(img, q[i], (32, 100), "resize"), ref)
        np.testing.assert_array_equal(C.host_crop(lib, img, q[i], (32, 100), "resize"), ref)


def test_golden(lib, optimized):
    """tests/golden/text_crop_ref.npz: the reference's own ImageCropper (oracle/make_text_crop_golden.py) on seeded images"""
    import os
    cv2.setUseOptimized(False)
    from oracle.make_text_crop_golden import CASES, case_inputs
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_crop_ref.npz"))
    for i, (name, dtype, mode, size) in enumerate(CASES):
        img, q, kinds = case_inputs(i, dtype)
        np.testing.assert_array_equal(g[name + "/quads"], q)
        geo = C.host_setup(lib, q, *img.shape[:2], mode, size)
        idx = g[name + "/index"]
        compared = 0
        for k in range(len(q)):
            crop = C.host_crop(lib, img, q[k], size, mode)
            if not _same_geometry(geo, k, q[k])[0]:        # the calipers class: cv2 through the product's matrix
                np.testing.assert_array_equal(crop, _cv2_crop(img, q[k], geo, k, size, mode, False), err_msg="%s %d" % (name, k))
                continue
            got = crop.reshape(-1)[idx]
            np.testing.assert_array_equal(got, g[name + "/plain"][k], err_msg="%s %d" % (name, k))
            np.testing.assert_array_equal(crop.astype(np.float64).sum((0, 1)), g[name + "/sums"][k], err_msg="%s %d" % (name, k))
            assert np.abs(got - g[name + "/default"][k]).max() <= DEFAULT_BOUND
            compared += 1
        assert compared >= len(q) // 2, name
