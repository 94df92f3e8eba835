"""The 256-pixel-tile convolution kernel, the weight-gradient plans and the row-split input gradient of csrc/conv_pingpong.cu.

- conv_fprop_m256_kernel (two 128-pixel tiles sharing one weight stage) must give the same bits as conv_fprop_tcgen05_kernel
  at every CRNN forward and input-gradient geometry that mr_conv_fprop_pp routes to it, and at the others when forced.
- mr_conv_wgrad_pp plans its splits from the CTA count it is given: the weight gradient must stay within
  tests.wgmma_variants.bound for CTA counts other than the 132 SMs of an H100 SXM (a PCIe card has 114).
- With a one-row dz (L6: 2 x 2 kernel, padding 0) the engine computes each input-gradient row as a 1 x 2 convolution with
  that row's taps, which must equal the 2 x 2 convolution over the padded dz."""
import re
import shutil

import pytest
import torch

from tests import wgmma_variants as wv
from tests.test_conv_pingpong_gpu import BATCHES, LAYERS, _crnn, _operands

M256_MIN_KB = 36          # kM256MinKb of csrc/conv_pingpong.cu


def k_blocks(lay, kind):
    """64-deep K blocks of the call: kh * kw * (input channels) / 64."""
    _, H, W, C, Cout, k, p = lay
    return k * k * (C if kind == "fprop" else Cout) // 64


def pixel_tiles(lay, kind, n):
    """128-pixel output tiles of plan_conv_segments (wgmma.cuh) for the call's output [n, Ho, Wo]."""
    _, H, W, C, Cout, k, p = lay
    Ho, Wo = (H + 2 * p - k + 1, W + 2 * p - k + 1) if kind == "fprop" else (H, W)
    tiles, w0 = 0, 0
    while w0 < Wo:
        bw = 128
        while bw > Wo - w0:
            bw //= 2
        bh = 1
        while bh * 2 <= Ho and bw * bh * 2 <= 128:
            bh *= 2
        bn = 128 // (bw * bh)
        nrep = (Wo - w0) // bw
        tiles += nrep * -(-Ho // bh) * -(-n // bn)
        w0 += nrep * bw
    return tiles


CASES = [(lay, kind, n) for lay in LAYERS for kind in ("fprop", "dgrad") for n in BATCHES]
SELECTED = [c for c in CASES if k_blocks(c[0], c[1]) >= M256_MIN_KB]
WGRAD_CTAS = [(lay, ctas) for lay in LAYERS for ctas in (132, 114, 100, 7)]


def test_cases_cover_odd_pixel_tile_counts():
    """The last pair of an odd tile count gives consumer 1 no tile; some selected cases must have one."""
    assert [c for c in SELECTED if pixel_tiles(*c) % 2 == 1]
    assert {(c[0][0], c[1]) for c in SELECTED} == {("L%d" % i, "fprop") for i in (3, 4, 5)} | \
        {("L%d" % i, "dgrad") for i in (2, 3, 4, 5)}


@pytest.mark.gpu
@pytest.mark.parametrize("lay,kind,n", CASES, ids=["%s-%s-N%d" % (c[0][0], c[1], c[2]) for c in CASES])
def test_m256_bit_identical_to_one_tile_kernel(cuda, lay, kind, n):
    """Forced onto the 256-pixel kernel (and, where the entry selects it, through the default selection too); L1's input
    gradient has 64 output channels, which that kernel does not take."""
    from megreader_b200 import nnops
    x, Wm, k, pad = _operands(lay, kind, n, cuda)
    want, Ho, Wo = nnops.conv_fprop_tc(x, Wm, k, k, pad, pad)
    if Wm.size(0) == 64:
        assert nnops.conv_fprop_pp(x, Wm, k, k, pad, pad, tile_m=256) is None
        return
    arms = [256] + ([0] if (lay, kind, n) in SELECTED else [])
    for tile_m in arms:
        r = nnops.conv_fprop_pp(x, Wm, k, k, pad, pad, tile_m=tile_m)
        assert r is not None, "conv_fprop_pp(tile_m=%d) refused a CRNN geometry" % tile_m
        got, Hp, Wp = r
        assert (Hp, Wp) == (Ho, Wo)
        diff = (got.float() - want.float()).abs()
        assert torch.equal(got, want), "tile_m=%d: %d of %d elements differ, worst %g" % (
            tile_m, int((diff > 0).sum()), diff.numel(), float(diff.max()))


@pytest.mark.gpu
def test_selection_by_k_blocks(cuda):
    """The entry takes the 256-pixel kernel from 36 K blocks on and the ping-pong kernel below (L6 forward: 32)."""
    from megreader_b200 import nnops
    for lay, kind in [(LAYERS[1], "fprop"), (LAYERS[1], "dgrad"), (LAYERS[0], "dgrad"), (LAYERS[5], "fprop")]:
        x, Wm, k, pad = _operands(lay, kind, 3, cuda)
        _, names = wv.launched_kernels(lambda: nnops.conv_fprop_pp(x, Wm, k, k, pad, pad))
        want = "conv_fprop_m256_kernel<128>" if k_blocks(lay, kind) >= M256_MIN_KB else "conv_fprop_pp_kernel<%d>" % (
            128 if Wm.size(0) > 64 else 64)
        assert names == {want}, (lay[0], kind, sorted(names))


@pytest.mark.gpu
@pytest.mark.parametrize("lay,ctas", WGRAD_CTAS, ids=["%s-ctas%d" % (c[0][0], c[1]) for c in WGRAD_CTAS])
def test_wgrad_plans_within_bound(cuda, lay, ctas):
    """N = 37 against float64 conv2d_weight on the same bf16 operands, with the grid capped at `ctas`."""
    from megreader_b200 import nnops
    _, H, W, C, Cout, k, p = lay
    n = 37
    g = torch.Generator(device=cuda).manual_seed(ctas * 13 + k)
    Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
    x = torch.randn((n, H, W, C), generator=g, device=cuda).bfloat16()
    dz = torch.randn((n, Ho, Wo, Cout), generator=g, device=cuda).bfloat16()
    got = nnops.conv_wgrad_pp(dz, x, k, k, p, p, ctas=ctas)
    assert got is not None, "conv_wgrad_pp refused a CRNN geometry"

    def ref(a, b):          # [Cout, k*k*C], columns (tap, channel) like the kernel's
        w = torch.nn.grad.conv2d_weight(a.double().permute(0, 3, 1, 2), (Cout, C, k, k), b.double().permute(0, 3, 1, 2),
                                        padding=p)
        return w.permute(0, 2, 3, 1).reshape(Cout, -1)
    wv.assert_within(got, ref(x, dz), wv.bound(ref(x.abs(), dz.abs())), "wgrad %s ctas=%d" % (lay[0], ctas))


@pytest.mark.gpu
@pytest.mark.parametrize("n", BATCHES)
def test_l6_row_split_dgrad_equals_the_padded_convolution(cuda, n):
    from megreader_b200 import crnn_engine
    lay = LAYERS[5]
    _, H, W, C, Cout, k, p = lay
    dz, Wd, _, _ = _operands(lay, "dgrad", n, cuda)
    want, _, _ = crnn_engine._conv_fprop(dz, Wd, k, k, k - 1 - p, k - 1 - p)
    got, names = wv.launched_kernels(lambda: crnn_engine._conv_dgrad(dz, Wd, k, k, p, p, H))
    assert got.shape == want.shape == (n * H * W, C)
    assert torch.equal(got, want)
    assert names == {"conv_fprop_pp_kernel<128>"}, sorted(names)     # 16 K blocks per row: the ping-pong kernel


@pytest.mark.gpu
def test_bf16_crnn_step_runs_the_m256_kernel(cuda):
    step = _crnn(cuda)
    step()
    _, names = wv.launched_kernels(step)
    assert "conv_fprop_m256_kernel<128>" in names, sorted(names)


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None,
                    reason="needs cuobjdump and cu++filt from the CUDA toolkit")
def test_every_m256_instantiation_has_a_gpu_case():
    from megreader_b200 import build
    from tests.test_kernel_inventory import compiled_kernels
    found = {n for n in map(wv.normalise, compiled_kernels(build.build())) if re.fullmatch(r"conv_fprop_m256_kernel<[\d,]+>", n)}
    assert found == {"conv_fprop_m256_kernel<128>"}, sorted(found)
