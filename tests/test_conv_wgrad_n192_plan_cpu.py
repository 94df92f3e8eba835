"""CPU: the schedule of the 128 x 192-tile weight gradient (mr_conv_wgrad_n192_plan, csrc/conv_pingpong.cu), which needs
no device.  It has the K-block plan of mr_conv_wgrad_pp_plan and counts ceil(Cout / 128) x ceil(K / 192) tiles; at L1 and
L2 the 192-column tiles cover K exactly, where the 256-column ones issue 768 and 1280 columns for K = 576 and 1152."""
import pytest

from tests.test_conv_wgrad_plan_cpu import MIN_KB, SMS, _check, _check_schedule

# (name, C, Cout, k, padding, Ho, Wo) of the CRNN layers the engine runs on 192-column tiles, and edge geometries
GEOMS = [("L1", 64, 128, 3, 1, 16, 128), ("L2", 128, 256, 3, 1, 8, 64), ("Cout192", 128, 192, 3, 1, 4, 65),
         ("K256", 64, 128, 2, 0, 2, 66), ("Wo80", 64, 64, 3, 1, 1, 80)]
NS = [1, 3, 37, 81, 512]


@pytest.fixture(scope="module")
def lib():
    from megreader_b200 import _lib, build
    build.build()
    return _lib


@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_n192_plan_tiles_and_schedule(lib, geom):
    from megreader_b200 import nnops
    _, C, Cout, k, p, Ho, Wo = geom
    H, W = Ho + k - 1 - 2 * p, Wo + k - 1 - 2 * p
    for N in NS:
        for ctas in (SMS, 7):
            plan = nnops.conv_wgrad_n192_plan(N, H, W, C, Cout, k, k, p, p, ctas, MIN_KB)
            pp = nnops.conv_wgrad_pp_plan(N, H, W, C, Cout, k, k, p, p, ctas, MIN_KB)
            assert plan["tiles"] == -(-Cout // 128) * -(-(k * k * C) // 192)
            assert (plan["RB"], plan["kb_total"], plan["segs"]) == (pp["RB"], pp["kb_total"], pp["segs"])
            _check(plan, N, Ho, Wo)
            _check_schedule(plan, ctas)


def test_n192_tiles_cover_k_exactly_at_l1_l2(lib):
    from megreader_b200 import nnops
    for C, Cout, tiles192, tiles256 in ((64, 128, 3, 3), (128, 256, 12, 10)):
        H, W = (16, 128) if C == 64 else (8, 64)
        n192 = nnops.conv_wgrad_n192_plan(512, H, W, C, Cout, 3, 3, 1, 1, SMS, MIN_KB)
        n256 = nnops.conv_wgrad_pp_plan(512, H, W, C, Cout, 3, 3, 1, 1, SMS, MIN_KB)
        assert (n192["tiles"], n256["tiles"]) == (tiles192, tiles256)
        # issued columns per 128-row block: K itself on 192-column tiles, 768 / 1280 on 256-column ones
        assert 192 * n192["tiles"] // -(-Cout // 128) == 9 * C
        assert 256 * n256["tiles"] // -(-Cout // 128) == {64: 768, 128: 1280}[C]
