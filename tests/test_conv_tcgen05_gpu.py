"""GPU: implicit-GEMM convolution kernels (wgmma + TMA + cp.async gather, csrc/gemm_tcgen05.cu) against PyTorch's
fp32 conv2d / autograd on bf16-rounded inputs."""
import zlib

import pytest
import torch
import torch.nn.functional as F

from tests import wgmma_variants as wv

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
    """large pixel counts on each activation path: the default TMA-A tiling with its shallow ring, the deep ring
    (MR_CONV_SHALLOW=0) and the cp.async gather (MR_CONV_NO_TMA_A=1); tiles that straddle a width-segment boundary in
    "bn64", a ragged last tile in "odd_tiles"."""
    from megreader_b200 import nnops
    N, H, W, C, Cout, k, p = geo
    torch.manual_seed(3)
    x = torch.randn(N, H, W, C, device=cuda).bfloat16()
    w = (torch.randn(Cout, C, k, k, device=cuda) / (C * k * k) ** 0.5).bfloat16()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), padding=p)
    for env in ({}, {"MR_CONV_SHALLOW": "0"}, {"MR_CONV_NO_TMA_A": "1"}):
        monkeypatch.delenv("MR_CONV_SHALLOW", raising=False)
        monkeypatch.delenv("MR_CONV_NO_TMA_A", raising=False)
        for key, val in env.items():
            monkeypatch.setenv(key, val)
        variant = wv.expected_variant("conv_fprop", H=H, W=W, Cout=Cout, kh=k, kw=k, ph=p, pw=p)
        y, Ho, Wo = wv.run_variant(variant, lambda: nnops.conv_fprop_tc(x, _wm(w), k, k, p, p, out_dtype=torch.float32))
        torch.testing.assert_close(y.view(N, Ho, Wo, Cout).permute(0, 3, 1, 2), ref, rtol=1e-3, atol=2e-3, msg=variant)


# ---------------------------------------------------------------- every instantiation, against float64 with an element-wise bound
def FP(N, H, W, C, Cout, k, s=1, p=0, d=1, out="f32", bias=False, relu=False, env=None, dgrad=False):
    """One forward case (square kernel k, stride s, padding p, dilation d); env: switches set for the call; dgrad: run
    the input-gradient form instead (x plays dz, flipped / transposed weights, padding k-1-p, stride 1)."""
    return dict(N=N, H=H, W=W, C=C, Cout=Cout, k=k, s=s, p=p, d=d, out=out, bias=bias, relu=relu, env=env or {},
                dgrad=dgrad)


FPROP = [
    # TMA-A tiling, shallow ring
    FP(2, 9, 17, 64, 128, 3, s=2, p=1), FP(3, 11, 13, 64, 38, 3, s=2, p=1),       # stride 2, odd H / W
    FP(2, 10, 20, 64, 38, 3, p=2, d=2), FP(1, 12, 24, 128, 96, 3, p=4, d=4),      # dilation 2 and 4
    FP(3, 8, 16, 64, 64, 1, s=2), FP(3, 2, 66, 64, 128, 2),                       # 1x1 stride 2; k = 2, p = 0
    FP(1, 2, 256, 64, 128, 3, p=1),                                               # Wo = 256: two 128-wide segments
    FP(2, 4, 15, 64, 64, 3, p=1),                                                 # Wo = 15: 8 + 4 + 2 + 1
    FP(9, 5, 7, 64, 128, 3, p=1),                                                 # several images per tile, ragged N
    # cp.async gather, reached by geometry: more than four segments, or a strided box wider than 256
    FP(2, 4, 31, 64, 38, 3, p=1), FP(2, 4, 31, 128, 128, 3, p=1),
    FP(1, 3, 300, 64, 64, 3, p=1), FP(1, 3, 300, 64, 192, 3, p=1),
    FP(1, 5, 390, 64, 64, 3, s=3, p=1), FP(2, 4, 384, 64, 128, 3, s=3, p=1),
    # switches: deep TMA-A ring, gather on a CRNN geometry
    FP(3, 16, 128, 64, 128, 3, p=1, env={"MR_CONV_SHALLOW": "0"}), FP(2, 8, 64, 128, 64, 3, p=1, env={"MR_CONV_SHALLOW": "0"}),
    FP(3, 16, 128, 64, 128, 3, p=1, env={"MR_CONV_NO_TMA_A": "1"}), FP(2, 8, 64, 128, 64, 3, p=1, env={"MR_CONV_NO_TMA_A": "1"}),
    # outputs: bf16, bias + ReLU, Cout = 1 and 38 (row pitch not 16-byte aligned: vector and scalar stores alternate)
    FP(2, 6, 10, 64, 128, 3, p=1, out="bf16", bias=True, relu=True), FP(2, 6, 10, 64, 38, 3, p=1, out="bf16"),
    FP(2, 6, 10, 64, 1, 3, p=1, bias=True, relu=True), FP(2, 4, 31, 64, 1, 3, p=1, out="bf16"),
    FP(2, 4, 31, 64, 38, 3, p=1, bias=True, relu=True), FP(1, 3, 300, 64, 200, 3, p=1, out="bf16", bias=True, relu=True),
    # input-gradient form on a TMA-A and a gather geometry
    FP(2, 8, 64, 128, 64, 3, p=1, dgrad=True), FP(2, 4, 31, 64, 128, 3, p=1, dgrad=True),
]


def _fp_id(c):
    s = "%dx%dx%dx%d-%d-k%ds%dp%dd%d" % (c["N"], c["H"], c["W"], c["C"], c["Cout"], c["k"], c["s"], c["p"], c["d"])
    s += "".join("-" + k for k in ("bias", "relu", "dgrad") if c[k]) + ("-bf16" if c["out"] == "bf16" else "")
    return s + "".join("-%s=%s" % kv for kv in sorted(c["env"].items()))


def fprop_variant(c):
    if c["dgrad"]:
        q = c["k"] - 1 - c["p"]
        return wv.expected_variant("conv_fprop", H=c["H"], W=c["W"], Cout=c["C"], kh=c["k"], kw=c["k"], ph=q, pw=q,
                                   env=c["env"])
    return wv.expected_variant("conv_fprop", H=c["H"], W=c["W"], Cout=c["Cout"], kh=c["k"], kw=c["k"], sh=c["s"],
                               sw=c["s"], ph=c["p"], pw=c["p"], dh=c["d"], dw=c["d"], env=c["env"])


def WG(N, H, W, C, Cout, k, s=1, p=0, d=1, splits=0):
    return dict(N=N, H=H, W=W, C=C, Cout=Cout, k=k, s=s, p=p, d=d, splits=splits)


WGRAD = [
    WG(2, 8, 64, 64, 128, 3, p=1), WG(2, 6, 72, 64, 64, 3, p=1),                 # <128,64,6>, <128,80,4>
    WG(3, 5, 40, 64, 40, 1), WG(2, 4, 72, 64, 192, 1),                           # <64,64,8>, <64,80,6> (1x1, C = 64)
    WG(2, 9, 33, 64, 64, 3, s=2, p=1), WG(2, 10, 30, 64, 128, 3, p=2, d=2),      # stride 2, dilation 2
    WG(2, 6, 20, 64, 8, 3, p=1), WG(2, 6, 20, 128, 40, 3, p=1), WG(1, 4, 100, 64, 192, 3, p=1),   # Cout 8 / 40 / 192
    WG(1, 4, 100, 64, 64, 3, p=1, splits=1), WG(2, 6, 72, 64, 64, 3, p=1, splits=10 ** 6),        # Wo = 100; splits
    WG(2, 4, 72, 64, 192, 1, splits=1), WG(3, 5, 40, 64, 40, 1, splits=10 ** 6),
]


def _wg_id(c):
    return "%dx%dx%dx%d-%d-k%ds%dp%dd%d-splits%d" % (c["N"], c["H"], c["W"], c["C"], c["Cout"], c["k"], c["s"], c["p"],
                                                     c["d"], c["splits"])


def wgrad_variant(c):
    return wv.expected_variant("conv_wgrad", H=c["H"], W=c["W"], C=c["C"], kh=c["k"], kw=c["k"], sh=c["s"], sw=c["s"],
                               ph=c["p"], pw=c["p"], dh=c["d"], dw=c["d"])


VARIANTS = {fprop_variant(c) for c in FPROP} | {wgrad_variant(c) for c in WGRAD}


def _nchw64(t):
    return t.double().permute(0, 3, 1, 2)


@pytest.mark.parametrize("c", FPROP, ids=[_fp_id(c) for c in FPROP])
def test_fprop_variant_vs_float64(cuda, c, monkeypatch):
    """conv2d_fprop_tc (stride, dilation, bias, ReLU, fp32 / bf16 out) and its input-gradient form against float64
    F.conv2d / conv2d_input on the same bf16 operands, element-wise within wv.bound."""
    from megreader_b200 import nnops
    monkeypatch.delenv("MR_CONV_SHALLOW", raising=False)
    monkeypatch.delenv("MR_CONV_NO_TMA_A", raising=False)
    for key, val in c["env"].items():
        monkeypatch.setenv(key, val)
    torch.manual_seed(zlib.crc32(_fp_id(c).encode()))
    N, H, W, C, Cout, k, s, p, d = (c[n] for n in ("N", "H", "W", "C", "Cout", "k", "s", "p", "d"))
    dtype = torch.bfloat16 if c["out"] == "bf16" else torch.float32
    w = torch.randn(Cout, C, k, k, device=cuda).bfloat16()
    bias = torch.randn(C if c["dgrad"] else Cout, device=cuda) if c["bias"] else None
    if c["dgrad"]:
        # dx[N,H,W,C] from dz[N,H+2p-k+1,...,Cout]: convolution with w flipped and transposed, padding k-1-p
        Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
        dz = torch.randn(N, Ho, Wo, Cout, device=cuda).bfloat16()
        wd = w.flip(2, 3).permute(1, 2, 3, 0).reshape(C, k * k * Cout).contiguous()
        q = k - 1 - p
        y, Hy, Wy = wv.run_variant(fprop_variant(c), lambda: nnops.conv2d_fprop_tc(dz, wd, k, k, 1, 1, q, q, 1, 1, dtype,
                                                                                 bias, c["relu"]))
        assert (Hy, Wy) == (H, W)
        ref = torch.nn.grad.conv2d_input((N, C, H, W), w.double(), _nchw64(dz), padding=p)
        absref = torch.nn.grad.conv2d_input((N, C, H, W), w.double().abs(), _nchw64(dz).abs(), padding=p)
        Co = C
    else:
        x = torch.randn(N, H, W, C, device=cuda).bfloat16()
        y, Hy, Wy = wv.run_variant(fprop_variant(c), lambda: nnops.conv2d_fprop_tc(x, _wm(w), k, k, s, s, p, p, d, d, dtype,
                                                                                 bias, c["relu"]))
        ref = F.conv2d(_nchw64(x), w.double(), None, s, p, d)
        absref = F.conv2d(_nchw64(x).abs(), w.double().abs(), None, s, p, d)
        Co = Cout
    assert ref.shape == (N, Co, Hy, Wy)
    if bias is not None:
        ref, absref = ref + bias.double().view(1, -1, 1, 1), absref + bias.double().abs().view(1, -1, 1, 1)
    if c["relu"]:
        ref = torch.relu(ref)
    got = y.view(N, Hy, Wy, Co).permute(0, 3, 1, 2)
    wv.assert_within(got, ref, wv.bound(absref, ref, dtype == torch.bfloat16), fprop_variant(c) + " " + _fp_id(c))


@pytest.mark.parametrize("c", WGRAD, ids=[_wg_id(c) for c in WGRAD])
def test_wgrad_variant_vs_float64(cuda, c):
    """conv2d_wgrad_tc against float64 conv2d_weight on the same bf16 operands, element-wise within wv.bound
    (fp32 atomics of the split-K partial sums included)."""
    from megreader_b200 import nnops
    torch.manual_seed(zlib.crc32(_wg_id(c).encode()))
    N, H, W, C, Cout, k, s, p, d = (c[n] for n in ("N", "H", "W", "C", "Cout", "k", "s", "p", "d"))
    Ho, Wo = wv.conv_out(H, W, k, k, s, s, p, p, d, d)
    x = torch.randn(N, H, W, C, device=cuda).bfloat16()
    dz = torch.randn(N, Ho, Wo, Cout, device=cuda).bfloat16()
    dWm = wv.run_variant(wgrad_variant(c), lambda: nnops.conv2d_wgrad_tc(dz, x, k, k, s, s, p, p, d, d, splits=c["splits"]))
    as_wm = lambda g: g.permute(0, 2, 3, 1).reshape(Cout, -1)  # noqa: E731
    ref = as_wm(torch.nn.grad.conv2d_weight(_nchw64(x), (Cout, C, k, k), _nchw64(dz), s, p, d))
    absref = as_wm(torch.nn.grad.conv2d_weight(_nchw64(x).abs(), (Cout, C, k, k), _nchw64(dz).abs(), s, p, d))
    wv.assert_within(dWm, ref, wv.bound(absref), wgrad_variant(c) + " " + _wg_id(c))
