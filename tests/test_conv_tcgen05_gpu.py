"""GPU: implicit-GEMM convolution kernels (wgmma + TMA + cp.async gather, csrc/gemm_tcgen05.cu) against PyTorch's
fp32 conv2d / autograd on bf16-rounded inputs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

GEOS = [  # N, H, W, C, Cout, k, pad       (CRNN layer geometries at small batch + edge cases)
    (3, 16, 128, 64, 128, 3, 1), (2, 8, 64, 128, 256, 3, 1), (2, 4, 65, 256, 512, 3, 1), (3, 2, 66, 512, 512, 2, 0),
    (5, 5, 7, 64, 64, 3, 1), (1, 9, 33, 128, 192, 3, 1),
]


def _wm(w):
    return w.permute(0, 2, 3, 1).reshape(w.size(0), -1).contiguous().bfloat16()


@pytest.mark.parametrize("geo", GEOS, ids=[str(i) for i in range(len(GEOS))])
def test_fprop_dgrad_wgrad(cuda, geo):
    from megreader_b200 import nnops
    N, H, W, C, Cout, k, p = geo
    torch.manual_seed(0)
    x = torch.randn(N, H, W, C, device=cuda).bfloat16()
    w = (torch.randn(Cout, C, k, k, device=cuda) / (C * k * k) ** 0.5).bfloat16()
    xr = x.float().permute(0, 3, 1, 2).requires_grad_(True)
    wr = w.float().requires_grad_(True)
    ref = F.conv2d(xr, wr, padding=p)
    y, Ho, Wo = nnops.conv_fprop_tc(x, _wm(w), k, k, p, p, out_dtype=torch.float32)
    torch.testing.assert_close(y.view(N, Ho, Wo, Cout).permute(0, 3, 1, 2), ref, rtol=1e-3, atol=2e-3)
    dz = torch.randn(N, Ho, Wo, Cout, device=cuda).bfloat16()
    ref.backward(dz.float().permute(0, 3, 1, 2))
    # input gradient = convolution of dz with flipped / transposed weights, padding k-1-p
    wd = w.flip(2, 3).permute(1, 2, 3, 0).reshape(C, k * k * Cout).contiguous()
    dx, Hb, Wb = nnops.conv_fprop_tc(dz, wd, k, k, k - 1 - p, k - 1 - p, out_dtype=torch.float32)
    assert (Hb, Wb) == (H, W)
    torch.testing.assert_close(dx.view(N, H, W, C).permute(0, 3, 1, 2), xr.grad, rtol=1e-3, atol=5e-3)
    dWm = nnops.conv_wgrad_tc(dz, x, k, k, p, p)
    refw = wr.grad.permute(0, 2, 3, 1).reshape(Cout, -1)
    torch.testing.assert_close(dWm, refw, rtol=1e-3, atol=2e-2 * (N * Ho * Wo) ** 0.5 / 10)


def test_fprop_bias_relu_bf16_out(cuda):
    from megreader_b200 import nnops
    torch.manual_seed(1)
    x = torch.randn(2, 6, 10, 64, device=cuda).bfloat16()
    w = (torch.randn(128, 64, 3, 3, device=cuda) / 24).bfloat16()
    b = torch.randn(128, device=cuda)
    y, Ho, Wo = nnops.conv_fprop_tc(x, _wm(w), 3, 3, 1, 1, bias=b, relu=True)
    ref = F.relu(F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, padding=1))
    torch.testing.assert_close(y.float().view(2, Ho, Wo, 128).permute(0, 3, 1, 2), ref, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("geo", [(40, 16, 128, 64, 128, 3, 1), (160, 8, 64, 128, 256, 3, 1), (300, 4, 65, 64, 64, 3, 1),
                                 (593, 1, 128, 64, 128, 3, 1)],
                         ids=["bn128", "bn256", "bn64", "odd_tiles"])
def test_fprop_large_p(cuda, geo, monkeypatch):
    """large pixel counts, once with the default one-tile CTAs and once with the two-tiles-per-CTA variant (MR_CONV_MT2=1):
    pairs that straddle a width-segment boundary in "bn64", an unpaired last tile in "odd_tiles"."""
    from megreader_b200 import nnops
    N, H, W, C, Cout, k, p = geo
    torch.manual_seed(3)
    x = torch.randn(N, H, W, C, device=cuda).bfloat16()
    w = (torch.randn(Cout, C, k, k, device=cuda) / (C * k * k) ** 0.5).bfloat16()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), padding=p)
    for mt2 in ("0", "1"):
        monkeypatch.setenv("MR_CONV_MT2", mt2)
        y, Ho, Wo = nnops.conv_fprop_tc(x, _wm(w), k, k, p, p, out_dtype=torch.float32)
        torch.testing.assert_close(y.view(N, Ho, Wo, Cout).permute(0, 3, 1, 2), ref, rtol=1e-3, atol=2e-3)
