"""GPU: the general wgmma convolution (stride, dilation, 1x1 / 3x3 / stem) behind megreader_b200.conv_engine against
torch's conv2d in fp32 on the same bf16-rounded operands -- forward, input gradient, weight gradient, bias gradient -- at the
geometries of the ResNet-50 / dilated / PPM / FPN trunks and the 2D-CTC head (SURVEY.md section 8 rows A4, A10)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

CASES = [
    # Cin, Cout, k, s, p, d, N, H, W, bias
    (64, 64, 1, 1, 0, 1, 2, 16, 64, False),      # bottleneck conv1
    (64, 256, 1, 1, 0, 1, 2, 16, 64, False),     # bottleneck conv3 / downsample
    (128, 128, 3, 2, 1, 1, 2, 16, 64, False),    # layer2.0.conv2 (stride 2)
    (256, 512, 1, 2, 0, 1, 2, 16, 64, False),    # layer2.0.downsample (1x1 stride 2)
    (256, 256, 3, 1, 2, 2, 2, 8, 32, False),     # dilated layer3
    (512, 512, 3, 1, 4, 4, 1, 8, 32, False),     # dilated layer4
    (256, 256, 3, 1, 1, 1, 3, 8, 32, True),      # CTCDecoder2D branch 3x3 (with bias)
    (256, 38, 1, 1, 0, 1, 3, 8, 32, True),       # classify 1x1
    (256, 1, 1, 1, 0, 1, 3, 8, 32, True),        # mask 1x1 (one output channel)
    (128, 128, 3, 2, 1, 1, 2, 15, 33, False),    # odd sizes under stride 2
    (64, 64, 3, 1, 1, 1, 2, 12, 65, True),       # width with a 1-wide TMA segment
    (3, 64, 7, 2, 3, 1, 2, 64, 96, False),       # stem (unfold + GEMM)
    (3, 64, 7, 2, 3, 1, 4, 128, 256, False),     # stem with enough pixels for the split-K weight gradient
]


@pytest.mark.parametrize("case", CASES, ids=[str(i) for i in range(len(CASES))])
def test_conv2d_forward_backward(cuda, case):
    from megreader_b200 import conv_engine
    Cin, Cout, k, s, p, d, N, H, W, with_bias = case
    torch.manual_seed(sum(case[:9]))
    x = torch.randn(N, Cin, H, W, device=cuda).bfloat16().float()
    w = (torch.randn(Cout, Cin, k, k, device=cuda) / (Cin * k * k) ** 0.5).bfloat16().float()
    b = torch.randn(Cout, device=cuda) if with_bias else None
    xr, wr = x.clone().requires_grad_(Cin % 64 == 0), w.clone().requires_grad_(True)
    br = b.clone().requires_grad_(True) if with_bias else None
    ref = F.conv2d(xr, wr, br, s, p, d)
    go = torch.randn_like(ref).bfloat16().float()
    ref.backward(go)
    conv = torch.nn.Conv2d(Cin, Cout, k, s, p, d, bias=with_bias).to(cuda)
    conv.weight.data.copy_(w)
    if with_bias:
        conv.bias.data.copy_(b)
    assert conv_engine.use_engine_convs(conv) == 1
    xe = x.clone().requires_grad_(Cin % 64 == 0)
    out = conv(xe)
    assert out.dtype == torch.bfloat16 and tuple(out.shape) == tuple(ref.shape)
    out.backward(go.to(out.dtype))

    def rel(a, r):
        return float((a.float() - r).norm() / (r.norm() + 1e-12))
    assert rel(out, ref) < 6e-3, rel(out, ref)
    assert rel(conv.weight.grad, wr.grad) < 1e-2, rel(conv.weight.grad, wr.grad)
    if with_bias:
        assert rel(conv.bias.grad, br.grad) < 1e-2
    if Cin % 64 == 0:
        assert rel(xe.grad, xr.grad) < 1e-2, rel(xe.grad, xr.grad)


def test_trunk_switch_counts_and_restores(cuda):
    from megreader_b200 import conv_engine
    m = torch.nn.Sequential(torch.nn.Conv2d(3, 64, 7, 2, 3), torch.nn.Conv2d(64, 64, 3, padding=1),
                            torch.nn.Conv2d(64, 32, 1), torch.nn.Conv2d(32, 32, 3, groups=2))
    assert conv_engine.use_engine_convs(m) == 3            # 32 -> 32 grouped stays with the library
    assert conv_engine.restore_library_convs(m) == 3
    with pytest.raises(NotImplementedError):
        conv_engine.conv2d(torch.zeros(1, 64, 4, 4), torch.zeros(64, 64, 1, 1))


BN_CASES = [
    # C, N, H, W, dtype, training
    (64, 4, 16, 64, torch.float32, True),
    (256, 4, 16, 64, torch.bfloat16, True),
    (2048, 8, 8, 32, torch.bfloat16, True),       # layer4 of the dilated trunk: 2 * C = 4096 statistic columns
    (1024, 3, 7, 9, torch.float32, True),         # odd row count
    (512, 4, 8, 32, torch.bfloat16, False),       # frozen statistics (eval with gradients)
    (64, 8, 128, 128, torch.bfloat16, True),      # 131,072 rows (the 512 x 512 scenes of the EAST configuration)
]


@pytest.mark.parametrize("case", BN_CASES, ids=[str(i) for i in range(len(BN_CASES))])
def test_batchnorm_forward_backward(cuda, case):
    """EngineBatchNorm2d (NHWC row kernels) against nn.BatchNorm2d in fp32 on the same (dtype-rounded) input: output, running
    statistics, input / weight / bias gradients"""
    from megreader_b200 import conv_engine
    C, N, H, W, dtype, training = case
    torch.manual_seed(C + N)
    x = (torch.randn(N, C, H, W, device=cuda) * 1.7 + 0.3).to(dtype).float()
    go = torch.randn(N, C, H, W, device=cuda).to(dtype).float()
    ref = torch.nn.BatchNorm2d(C).to(cuda)
    with torch.no_grad():
        ref.weight.copy_(torch.rand(C, device=cuda) + 0.5)
        ref.bias.copy_(torch.randn(C, device=cuda))
        ref.running_mean.copy_(0.1 * torch.randn(C, device=cuda))
        ref.running_var.copy_(torch.rand(C, device=cuda) + 0.5)
    eng = torch.nn.BatchNorm2d(C).to(cuda)
    eng.load_state_dict(ref.state_dict())
    wrap = torch.nn.Sequential(eng)
    conv_engine.use_engine_convs(wrap)
    assert type(wrap[0]) is conv_engine.EngineBatchNorm2d
    ref.train(training)
    wrap.train(training)
    xr = x.clone().requires_grad_(True)
    yr = ref(xr)
    yr.backward(go)
    xe = x.to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    ye = wrap(xe)
    assert ye.dtype == dtype and tuple(ye.shape) == (N, C, H, W)
    ye.backward(go.to(dtype))
    tol = 2e-5 if dtype == torch.float32 else 6e-3

    def rel(a, r):
        return float((a.float() - r).norm() / (r.norm() + 1e-12))
    assert rel(ye, yr) < tol, rel(ye, yr)
    assert rel(xe.grad, xr.grad) < 2 * tol, rel(xe.grad, xr.grad)
    assert rel(eng.weight.grad, ref.weight.grad) < 2 * tol and rel(eng.bias.grad, ref.bias.grad) < 2 * tol
    assert rel(eng.running_mean, ref.running_mean) < 1e-5 and rel(eng.running_var, ref.running_var) < 1e-5
    assert int(eng.num_batches_tracked) == int(ref.num_batches_tracked)
    assert conv_engine.restore_library_convs(wrap) == 0 and type(wrap[0]) is torch.nn.BatchNorm2d


@pytest.mark.parametrize("case", [(256, 128, 2, 16, 24, True), (128, 64, 1, 9, 7, False)], ids=["256-128", "128-64-odd"])
def test_conv_transpose_2x2(cuda, case):
    """EngineConvTranspose2d (kernel = stride = 2: a 1x1 engine convolution to 4 C_out channels + depth-to-space) against
    F.conv_transpose2d in fp32 on the same bf16-rounded operands (decoders/east.py:20-21)"""
    from megreader_b200 import conv_engine
    cin, cout, n, h, w, with_bias = case
    torch.manual_seed(cin + cout)
    x = torch.randn(n, cin, h, w, device=cuda).bfloat16().float()
    m = torch.nn.ConvTranspose2d(cin, cout, 2, 2, bias=with_bias).to(cuda)
    m.weight.data = m.weight.data.bfloat16().float()
    xr = x.clone().requires_grad_(True)
    ref = F.conv_transpose2d(xr, m.weight, m.bias, 2)
    go = torch.randn_like(ref).bfloat16().float()
    gw_ref, gb_ref = torch.autograd.grad(ref, [m.weight] + ([m.bias] if with_bias else []), go, retain_graph=True) if with_bias else \
        (torch.autograd.grad(ref, [m.weight], go, retain_graph=True)[0], None)
    gx_ref = torch.autograd.grad(ref, xr, go)[0]
    wrap = torch.nn.Sequential(m)
    conv_engine.use_engine_convs(wrap)
    assert type(wrap[0]) is conv_engine.EngineConvTranspose2d
    xe = x.clone().requires_grad_(True)
    out = wrap(xe)
    assert tuple(out.shape) == tuple(ref.shape)
    out.backward(go.to(out.dtype))

    def rel(a, r):
        return float((a.float() - r).norm() / (r.norm() + 1e-12))
    assert rel(out, ref) < 6e-3, rel(out, ref)
    assert rel(xe.grad, gx_ref) < 1e-2 and rel(m.weight.grad, gw_ref) < 1e-2
    if with_bias:
        assert rel(m.bias.grad, gb_ref) < 1e-2
    conv_engine.restore_library_convs(wrap)
    assert type(wrap[0]) is torch.nn.ConvTranspose2d
