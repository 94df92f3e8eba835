"""The persistent weight gradient's dense K blocks (csrc/conv_pingpong.cu, plan_wgrad_segments): for 64 < Wo <= 80 a K
block is 80 pixels in boxes of bw columns x 1 row x (80 / bw) images, cut from up to five column segments, each with its
own dz and x tensor maps.  Against float64 conv2d_weight on the same bf16 operands within tests.wgmma_variants.bound at
the edges of the plan (every Wo the CPU plan test covers, 3x3 / pad 1 and 2x2 / pad 0, batches that leave remainders in
the 5- and 80-image boxes), and at the six CRNN geometries at N = 512 against conv_wgrad_tcgen05_kernel within twice the
bound, with the instantiation each call means."""
import pytest
import torch

from tests import wgmma_variants as wv

# (name, input H, W, C, Cout, k, padding) of the implicit convolutions of backbones/crnn.py at 32 x 256 lines
LAYERS = [("L1", 16, 128, 64, 128, 3, 1), ("L2", 8, 64, 128, 256, 3, 1), ("L3", 8, 64, 256, 256, 3, 1),
          ("L4", 4, 65, 256, 512, 3, 1), ("L5", 4, 65, 512, 512, 3, 1), ("L6", 2, 66, 512, 512, 2, 0)]
# (k, padding, Ho) x Wo x N: Cout = 192 leaves half a 128-row tile, K = 9 * 128 or 4 * 128 a partial 256-column tile
EDGE = [(k, p, Ho, Wo, n) for k, p, hos in ((3, 1, (1, 4)), (2, 0, (1, 2))) for Ho in hos for Wo in (65, 66, 72, 79, 80)
        for n in (3, 5, 37, 81)]


def _kernel(Wo):
    return "conv_wgrad_pp_kernel<%d>" % (80 if 64 < Wo <= 80 else 64)


def _ref(x, dz, Cout, C, k, p):
    """float64 conv2d_weight as [Cout, k*k*C], columns (tap, channel) like the kernel's"""
    w = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (Cout, C, k, k), dz.double().permute(0, 3, 1, 2),
                                    padding=p)
    return w.permute(0, 2, 3, 1).reshape(Cout, -1)


@pytest.mark.gpu
@pytest.mark.parametrize("k,p,Ho,Wo,n", EDGE, ids=["k%d-Ho%d-Wo%d-N%d" % (c[0], c[2], c[3], c[4]) for c in EDGE])
def test_dense_wgrad_edges_within_bound(cuda, k, p, Ho, Wo, n):
    from megreader_b200 import nnops
    C, Cout = 128, 192
    H, W = Ho + k - 1 - 2 * p, Wo + k - 1 - 2 * p
    g = torch.Generator(device=cuda).manual_seed(1000 * Wo + 10 * n + k)
    x = torch.randn((n, H, W, C), generator=g, device=cuda).bfloat16()
    dz = torch.randn((n, Ho, Wo, Cout), generator=g, device=cuda).bfloat16()
    got = nnops.conv_wgrad_pp(dz, x, k, k, p, p)
    assert got is not None, "conv_wgrad_pp refused the geometry"
    wv.assert_within(got, _ref(x, dz, Cout, C, k, p), wv.bound(_ref(x.abs(), dz.abs(), Cout, C, k, p)),
                     "wgrad k=%d Ho=%d Wo=%d N=%d" % (k, Ho, Wo, n))


@pytest.mark.gpu
@pytest.mark.parametrize("lay", LAYERS, ids=[x[0] for x in LAYERS])
def test_dense_wgrad_crnn_layers_against_one_tile_kernel(cuda, lay):
    from megreader_b200 import nnops
    name, H, W, C, Cout, k, p = lay
    n = 512
    Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
    g = torch.Generator(device=cuda).manual_seed(17 * k + C)
    x = torch.randn((n, H, W, C), generator=g, device=cuda).bfloat16()
    dz = torch.randn((n, Ho, Wo, Cout), generator=g, device=cuda).bfloat16()
    got, names = wv.launched_kernels(lambda: nnops.conv_wgrad_pp(dz, x, k, k, p, p))
    assert got is not None, "conv_wgrad_pp refused a CRNN geometry"
    ours = sorted(nm for nm in names if nm.startswith("conv_wgrad_pp_kernel"))
    if ours or any(nm.startswith("conv_") for nm in names):     # a trace with no library kernel says nothing
        assert ours == [_kernel(Wo)], sorted(names)
    want = nnops.conv_wgrad_tc(dz, x, k, k, p, p)
    bnd = 2 * wv.bound(nnops.conv_wgrad_tc(dz.abs(), x.abs(), k, k, p, p).double())
    wv.assert_within(got, want, bnd, "wgrad %s N=%d" % (name, n))
