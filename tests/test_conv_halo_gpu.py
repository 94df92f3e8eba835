"""The halo mode of the ping-pong convolution (csrc/conv_pingpong.cu, conv_fprop_pp_kernel): where every pixel tile is one
whole 128-pixel output row, the kernel loads one (128 + kw - 1)-pixel activation halo per (tap row, channel block) and runs
the row's kw taps from it, with the A descriptor j rows into the halo.  K order and instruction sequence are unchanged, so
the output must be torch.equal to conv_fprop_tcgen05_kernel's at every geometry the mode takes: 3x3 / pad 1 and 2x2 /
pad 0, C = 64, 128 and (2x2) 256 (one to four live halo slots per tap row), Cout = 64 and 128 (BN = 64, 128), output rows of 128
and 256 pixels (one and two segments), N = 1, 3, 37 and 512.  nnops.conv_fprop_pp_halo (host only) says which calls take
the mode; it is checked on the CPU against the CRNN layers: L1's forward and input gradient, nothing else."""
import pytest
import torch

# (k, padding, C, Cout, Wo, N)
CASES = [(k, p, C, Cout, Wo, n) for k, p in ((3, 1), (2, 0)) for C in (64, 128, 256) for Cout in (64, 128)
         for Wo in (128, 256) for n in ((1, 3, 37, 512) if Wo == 128 else (1, 37))
         if k * k * C // 64 < 36]                    # from 36 K blocks on the 256-pixel kernel runs instead
# (name, input H, W, C, Cout, k, padding) of the implicit convolutions of backbones/crnn.py at 32 x 256 lines
LAYERS = [("L1", 16, 128, 64, 128, 3, 1), ("L2", 8, 64, 128, 256, 3, 1), ("L3", 8, 64, 256, 256, 3, 1),
          ("L4", 4, 65, 256, 512, 3, 1), ("L5", 4, 65, 512, 512, 3, 1), ("L6", 2, 66, 512, 512, 2, 0)]


@pytest.fixture(scope="module")
def lib():
    from megreader_b200 import _lib, build
    build.build()
    return _lib


@pytest.mark.gpu
@pytest.mark.parametrize("k,p,C,Cout,Wo,n", CASES, ids=["k%d-C%d-Cout%d-Wo%d-N%d" % ((c[0],) + c[2:]) for c in CASES])
def test_halo_mode_bit_identical_to_one_tile_kernel(cuda, k, p, C, Cout, Wo, n):
    from megreader_b200 import nnops
    Ho = 4
    H, W = Ho + k - 1 - 2 * p, Wo + k - 1 - 2 * p
    assert nnops.conv_fprop_pp_halo(H, W, C, Cout, k, k, p, p)
    g = torch.Generator(device=cuda).manual_seed(1000 * C + 10 * n + k + Cout)
    x = torch.randn((n, H, W, C), generator=g, device=cuda).bfloat16()
    Wm = (torch.randn((Cout, k * k * C), generator=g, device=cuda) / (k * k * C) ** 0.5).bfloat16()
    want, _, _ = nnops.conv_fprop_tc(x, Wm, k, k, p, p)
    got = nnops.conv_fprop_pp(x, Wm, k, k, p, p)
    assert got is not None, "conv_fprop_pp refused the geometry"
    assert torch.equal(got[0], want), "halo mode differs from conv_fprop_tc: max |diff| %g" % float(
        (got[0].float() - want.float()).abs().max())


def test_halo_mode_takes_l1_forward_and_input_gradient_only(lib):
    from megreader_b200 import nnops
    took = set()
    for name, H, W, C, Cout, k, p in LAYERS:
        if nnops.conv_fprop_pp_halo(H, W, C, Cout, k, k, p, p):
            took.add((name, "fprop"))
        if nnops.conv_fprop_pp_halo(H + 2 * p - k + 1, W + 2 * p - k + 1, Cout, C, k, k, k - 1 - p, k - 1 - p):
            took.add((name, "dgrad"))
    assert took == {("L1", "fprop"), ("L1", "dgrad")}, sorted(took)


def test_halo_mode_geometry_limits(lib):
    from megreader_b200 import nnops
    assert nnops.conv_fprop_pp_halo(4, 128, 64, 64, 3, 3, 1, 1)
    assert not nnops.conv_fprop_pp_halo(4, 128, 64, 64, 3, 1, 1, 0)          # kw = 1: nothing to share
    assert not nnops.conv_fprop_pp_halo(4, 128, 320, 64, 3, 3, 1, 1)         # five channel blocks
    assert not nnops.conv_fprop_pp_halo(4, 192, 64, 64, 3, 3, 1, 1)          # a 64-wide segment
    assert not nnops.conv_fprop_pp_halo(4, 640, 64, 64, 3, 3, 1, 1)          # five segments
    assert not nnops.conv_fprop_pp_halo(4, 128, 256, 128, 3, 3, 1, 1)        # 36 K blocks: the 256-pixel kernel
    with pytest.raises(Exception):
        nnops.conv_fprop_pp_halo(4, 128, 64, 64, 3, 3, -1, 1)
