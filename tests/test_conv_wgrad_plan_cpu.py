"""CPU: the K-block plan of the persistent weight gradient (mr_conv_wgrad_pp_plan, csrc/conv_pingpong.cu), which needs no
device.  Every output pixel must lie in exactly one K-block box, the boxes of 64 < Wo <= 80 must hold real pixels only
(apart from a segment's last image block), the K-block count must be the plan's formula, and every CTA must get the same
number of (split, tile) units whenever the plan says it does."""
import numpy as np
import pytest

# (name, C, Cout, k, padding) of the implicit convolutions of backbones/crnn.py
LAYERS = [("L1", 64, 128, 3, 1), ("L2", 128, 256, 3, 1), ("L3", 256, 256, 3, 1), ("L4", 256, 512, 3, 1),
          ("L5", 512, 512, 3, 1), ("L6", 512, 512, 2, 0)]
WOS = [65, 66, 72, 79, 80]
HOS = [1, 2, 4]
NS = [1, 3, 5, 37, 80, 81, 512]
SMS = 132          # H100 SXM
MIN_KB = 16        # nnops._WGRAD_MIN_KB's default


@pytest.fixture(scope="module")
def lib():
    from megreader_b200 import _lib, build
    build.build()
    return _lib


def _plan(N, Ho, Wo, C, Cout, k, p, ctas):
    from megreader_b200 import nnops
    return nnops.conv_wgrad_pp_plan(N, Ho + k - 1 - 2 * p, Wo + k - 1 - 2 * p, C, Cout, k, k, p, p, ctas, MIN_KB)


def _formula(N, Ho, Wo):
    """K blocks of the plan: 16 x 1 x 5 boxes over the first Wo // 16 * 16 columns, then one bw x 1 x (80 / bw) box column
    for each power of two bw in Wo % 16; 64 < Wo <= 80 only, one 64-wide box per row otherwise."""
    if 64 < Wo <= 80:
        return Wo // 16 * Ho * -(-N // 5) + sum(Ho * -(-N // (80 // bw)) for bw in (8, 4, 2, 1) if Wo % 16 & bw)
    return -(-Wo // 64) * Ho * N


def _boxes(plan, Ho):
    """Every K block's box, decoded as the kernel's producer does: (segment, w, ho, n0) arrays."""
    segs = np.array(plan["segs"])
    kb = np.arange(plan["kb_total"])
    sel = np.searchsorted(segs[:, 4], kb, side="right") - 1
    w0, bw, bn, wbl, beg = (segs[sel, i] for i in range(5))
    r = kb - beg
    wb, r = r % wbl, r // wbl
    return sel, w0 + wb * bw, r % Ho, r // Ho * bn


def _check(plan, N, Ho, Wo):
    RB = plan["RB"]
    assert RB == (80 if 64 < Wo <= 80 else 64)
    segs = np.array(plan["segs"])
    assert 1 <= len(segs) <= 5 and segs[0, 0] == 0 and segs[0, 4] == 0
    assert np.all(segs[:, 1] * segs[:, 2] == RB), plan["segs"]
    assert plan["kb_total"] == _formula(N, Ho, Wo)
    sel, w, ho, n0 = _boxes(plan, Ho)
    bw, bn = segs[sel, 1], segs[sel, 2]
    assert np.all(n0 < N) and np.all(ho < Ho) and np.all(w < Wo)
    if RB == 80:
        assert np.all(w + bw <= Wo), "a box reaches past the output width"
    j = np.arange(RB)[None, :]
    pw = w[:, None] + j % bw[:, None]
    pn = n0[:, None] + j // bw[:, None]
    ph = np.broadcast_to(ho[:, None], pw.shape)
    real = (pw < Wo) & (pn < N)
    count = np.bincount(((pn * Ho + ph) * Wo + pw)[real], minlength=N * Ho * Wo)
    assert count.size == N * Ho * Wo and np.all(count == 1), "pixels in %s boxes" % sorted(set(count.tolist()))
    if RB == 80:                 # real pixels: all of them but the batch remainder of each segment's last image block
        pad = sum(s[3] * Ho * (-(-N // s[2]) * s[2] - N) * s[1] for s in plan["segs"])
        assert int((~real).sum()) == pad


def _check_schedule(plan, ctas):
    grid, units, tiles = plan["grid"], plan["units"], plan["tiles"]
    assert 1 <= grid <= ctas and units % tiles == 0
    splits = units // tiles
    assert plan["kb_split"] == -(-plan["kb_total"] // splits)
    if plan["balanced"]:
        per_cta = np.bincount(np.arange(units) % grid, minlength=grid)
        assert np.all(per_cta == per_cta[0]), "the plan claims equal units per CTA: %s" % sorted(set(per_cta.tolist()))
        assert grid * 10 >= 9 * min(ctas, plan["kb_total"] * tiles)


@pytest.mark.parametrize("lay", LAYERS, ids=[x[0] for x in LAYERS])
def test_wgrad_plan_boxes_and_schedule(lib, lay):
    _, C, Cout, k, p = lay
    for Wo in WOS:
        for Ho in HOS:
            for N in NS:
                plan = _plan(N, Ho, Wo, C, Cout, k, p, SMS)
                _check(plan, N, Ho, Wo)
                _check_schedule(plan, SMS)
                # the grid nnops.conv_wgrad_pp asks for by default
                ctas = min(SMS, max(1, plan["kb_total"] * plan["tiles"] // MIN_KB))
                _check_schedule(_plan(N, Ho, Wo, C, Cout, k, p, ctas), ctas)


@pytest.mark.parametrize("Wo", [1, 32, 64, 81, 128, 200])
def test_wgrad_plan_outside_the_dense_range_keeps_row_boxes(lib, Wo):
    """Wo <= 64 or > 80: one segment of 64-wide row boxes, as before the plan."""
    for Ho, N in ((1, 3), (4, 37)):
        plan = _plan(N, Ho, Wo, 256, 512, 3, 1, SMS)
        assert plan["segs"] == [(0, 64, 1, -(-Wo // 64), 0)]
        _check(plan, N, Ho, Wo)
        _check_schedule(plan, SMS)


def test_wgrad_plan_l5_is_dense(lib):
    """L5 at the bench batch: 1,676 K blocks of 80 pixels (99.3 % real) instead of 2,048 80-wide row boxes."""
    plan = _plan(512, 4, 65, 512, 512, 3, 1, SMS)
    assert plan["kb_total"] == 1676
    assert plan["segs"] == [(0, 16, 5, 4, 0), (64, 1, 80, 1, 1648)]
    assert round(512 * 4 * 65 / (plan["kb_total"] * 80), 3) == 0.993


def test_wgrad_plan_refuses_bad_arguments(lib):
    import ctypes
    plan = (ctypes.c_int * 33)()
    L = lib.lib()
    assert L.mr_conv_wgrad_pp_plan(4, 4, 65, 64, 128, 3, 3, 1, 1, 0, 16, plan) == 4      # MR_ERR_BAD_SHAPE: ctas < 1
    assert L.mr_conv_wgrad_pp_plan(4, 4, 65, 64, 128, 3, 3, 1, 1, 132, 16, None) == 1   # MR_ERR_NULL_POINTER
