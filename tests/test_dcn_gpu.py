"""GPU parity: deformable conv v1/v2 (sm_90a kernels + cuBLAS fp32 GEMM through the C-ABI) against the CPU oracle
(oracle/dcn_oracle.c, float64) on the same seeded inputs, including the reference's stride-2 offset quirk."""
import numpy as np
import pytest
import torch

from oracle import capi
from tests import wgmma_variants as wv

pytestmark = pytest.mark.gpu

CASES = [
    # B, C, H, W, Cout, k, stride, pad, dil, group, dg, modulated, bias
    (2, 4, 7, 9, 6, 3, 1, 1, 1, 1, 1, True, False),
    (2, 4, 8, 8, 4, 3, 2, 1, 1, 1, 1, True, True),
    (1, 8, 6, 5, 8, 3, 1, 1, 1, 2, 2, True, True),
    (2, 6, 9, 7, 4, 3, 1, 2, 2, 1, 3, True, False),
    (3, 4, 5, 5, 2, 1, 1, 0, 1, 1, 1, True, True),
    (8, 128, 16, 16, 128, 3, 1, 1, 1, 1, 1, True, False),   # Bottleneck-like (layer2 channels, small map)
    (2, 4, 7, 9, 6, 3, 1, 1, 1, 1, 1, False, False),         # DCNv1
    (4, 8, 6, 6, 4, 3, 1, 1, 1, 2, 1, False, False),         # DCNv1 grouped
    (2, 64, 13, 19, 128, 3, 2, 1, 1, 1, 1, True, True),      # fused wgmma forward + weight gradient: stride 2, ragged tiles
    (2, 128, 13, 19, 128, 3, 2, 1, 1, 1, 1, True, True),     # + fused data gradient (C % 128 == 0)
    (1, 256, 11, 18, 128, 3, 1, 1, 1, 1, 1, True, False),    # two 128-channel chunks per tap, ragged tiles
    (3, 128, 9, 21, 128, 3, 1, 2, 2, 1, 1, False, False),    # fused path, DCNv1 (no mask), dilation 2
]


def _inputs(seed, B, C, H, W, Cout, k, s, p, d, group, dg, big_offset=False):
    rng = np.random.RandomState(seed)
    Ho = (H + 2 * p - (d * (k - 1) + 1)) // s + 1
    Wo = (W + 2 * p - (d * (k - 1) + 1)) // s + 1
    oh, ow = (H, W) if big_offset else (Ho, Wo)
    x = rng.standard_normal((B, C, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, C // group, k, k)) * (1.0 / np.sqrt(C * k * k))).astype(np.float32)
    b = rng.standard_normal((Cout,)).astype(np.float32)
    off = (rng.standard_normal((B, 2 * k * k * dg, oh, ow)) * 1.5).astype(np.float32)
    m = (1 / (1 + np.exp(-rng.standard_normal((B, k * k * dg, oh, ow))))).astype(np.float32)
    go = rng.standard_normal((B, Cout, Ho, Wo)).astype(np.float32)
    return x, w, b, off, m, go


def _close(a, ref, what):
    scale = max(1.0, float(np.abs(ref).max()))
    np.testing.assert_allclose(a, ref, rtol=1e-4, atol=1e-4 * scale, err_msg=what)


@pytest.mark.parametrize("case", CASES, ids=[str(i) for i in range(len(CASES))])
def test_dcn_forward_backward_vs_oracle(cuda, case):
    from megreader_b200 import dcn
    B, C, H, W, Cout, k, s, p, d, group, dg, modulated, with_bias = case
    x, w, b, off, m, go = _inputs(1, B, C, H, W, Cout, k, s, p, d, group, dg)
    f64 = lambda a: a.astype(np.float64)  # noqa: E731
    o_ref = capi.dcn_forward(f64(x), f64(w), f64(b) if with_bias else None, f64(off), f64(m) if modulated else None,
                             s, p, d, group, dg)
    g_ref = capi.dcn_backward(f64(x), f64(w), f64(b) if with_bias else None, f64(off), f64(m) if modulated else None,
                              f64(go), s, p, d, group, dg)
    tx, tw, tb, toff, tm = [torch.from_numpy(a).to(cuda).requires_grad_(True) for a in (x, w, b, off, m)]
    if modulated:
        out = dcn.modulated_deform_conv(tx, toff, tm, tw, tb if with_bias else None, s, p, d, group, dg)
    else:
        out = dcn.deform_conv(tx, toff, tw, s, p, d, group, dg)
    _close(out.detach().cpu().numpy(), o_ref, "output")
    out.backward(torch.from_numpy(go).to(cuda))
    _close(tx.grad.cpu().numpy(), g_ref[0], "grad_input")
    _close(tw.grad.cpu().numpy(), g_ref[1], "grad_weight")
    _close(toff.grad.cpu().numpy(), g_ref[3], "grad_offset")
    if modulated:
        _close(tm.grad.cpu().numpy(), g_ref[4], "grad_mask")
    if with_bias:
        _close(tb.grad.cpu().numpy(), g_ref[2], "grad_bias")


FUSED_FWD_CASE = 8      # stride 2, ragged tiles: the fused wgmma forward


def test_dcn_fused_forward_rings(cuda):
    """the fused forward runs its one instantiation (the two-stage ring)."""
    wv.run_variant(wv.expected_variant("dcn_fwd"), lambda: test_dcn_forward_backward_vs_oracle(cuda, CASES[FUSED_FWD_CASE]))


VARIANTS = {wv.expected_variant("dcn_fwd")}


@pytest.mark.parametrize("dt", [torch.float32, torch.float16, torch.bfloat16], ids=["fp32", "fp16", "bf16"])
def test_dcn_fused_backward_unaligned_grad_output(cuda, dt):
    """grad_output a contiguous view one element into a larger buffer, so not 16-byte aligned: the fused backward gives the
    gradients of an aligned copy, bit for bit.  Wo = 16 is one whole tile row, so the aligned call re-tiles grad_output with
    16-byte loads.  A 3 x 3 kernel at stride 3 with zero offsets samples every input pixel once, and B = 1 with Ho = 8 is one
    pixel tile (one weight-gradient split), so every atomic sum has one term and the gradients are deterministic."""
    from megreader_b200 import dcn
    B, C, H, W, Cout, k, s = 1, 128, 24, 48, 128, 3, 3
    Ho, Wo = H // s, W // s
    gen = torch.Generator().manual_seed(11)
    rnd = lambda *shape, scale=1.0: (torch.randn(*shape, generator=gen) * scale).to(cuda, dt)  # noqa: E731
    x, w, b = rnd(B, C, H, W), rnd(Cout, C, k, k, scale=(C * k * k) ** -0.5), rnd(Cout)
    off = torch.zeros(B, 2 * k * k, Ho, Wo, device=cuda, dtype=dt)
    m = torch.sigmoid(rnd(B, k * k, Ho, Wo))
    go = rnd(B, Cout, Ho, Wo)
    buf = torch.empty(go.numel() + 1, device=cuda, dtype=dt)
    go_view = buf[1:].view(go.shape)
    go_view.copy_(go)
    assert go_view.is_contiguous() and go_view.data_ptr() % 16 != 0 and go.data_ptr() % 16 == 0

    def grads(grad_output):
        g = [torch.zeros_like(t) for t in (x, w, b, off, m)]
        dcn.modulated_deform_conv_cuda_backward(x, w, b, None, off, m, None, *g, grad_output, k, k, s, s, 0, 0, 1, 1, 1, 1,
                                                True)
        torch.cuda.synchronize()
        return g

    want, got = grads(go), grads(go_view)
    for name, a, e in zip(("grad_input", "grad_weight", "grad_bias", "grad_offset", "grad_mask"), got, want):
        assert e.abs().sum() > 0, name
        assert torch.equal(a, e), name


def test_dcn_stride2_offset_slice_quirk(cuda):
    """backbones/resnet.py:136-165: offset = offset_mask[:, :18] (non-contiguous batch slice, spatial size = INPUT
    size) with a stride-2 DCN -> per-sample slabs are re-read flat with (Ho,Wo) strides (App. B2.1)."""
    from megreader_b200 import dcn
    B, C, H, W, Cout, k, s, p = 3, 8, 8, 8, 8, 3, 2, 1
    x, w, _, _, _, go = _inputs(5, B, C, H, W, Cout, k, s, p, 1, 1, 1)
    rng = np.random.RandomState(9)
    offset_mask = rng.standard_normal((B, 27, H, W)).astype(np.float32)
    tom = torch.from_numpy(offset_mask).to(cuda).requires_grad_(True)
    tx, tw = [torch.from_numpy(a).to(cuda).requires_grad_(True) for a in (x, w)]
    offset = tom[:, :18, :, :]
    mask = tom[:, -9:, :, :].sigmoid()
    assert not offset.is_contiguous()
    out = dcn.modulated_deform_conv(tx, offset, mask, tw, None, s, p, 1, 1, 1)
    off_np = offset_mask[:, :18]
    m_np = 1 / (1 + np.exp(-offset_mask[:, -9:].astype(np.float64)))
    o_ref = capi.dcn_forward(x.astype(np.float64), w.astype(np.float64), None, off_np.astype(np.float64), m_np, s, p, 1)
    _close(out.detach().cpu().numpy(), o_ref, "output")
    out.backward(torch.from_numpy(go).to(cuda))
    gi, gw, _, goff, gm = capi.dcn_backward(x.astype(np.float64), w.astype(np.float64), None,
                                            off_np.astype(np.float64), m_np, go.astype(np.float64), s, p, 1)
    _close(tx.grad.cpu().numpy(), gi, "grad_input")
    _close(tw.grad.cpu().numpy(), gw, "grad_weight")
    ref_gom = np.concatenate([goff, gm * m_np * (1 - m_np)], axis=1)    # chain through sigmoid for the mask part
    _close(tom.grad.cpu().numpy(), ref_gom, "grad offset_mask")


def test_dcn_pybind_surface_in_place(cuda):
    """modulated_deform_conv_cuda_forward writes the caller's `output` in place and accumulates into caller-zeroed
    grads (functions/deform_conv.py:135-160)."""
    from megreader_b200 import dcn
    x, w, b, off, m, go = _inputs(2, 2, 4, 6, 6, 4, 3, 1, 1, 1, 1, 1)
    tx, tw, tb, toff, tm, tgo = [torch.from_numpy(a).to(cuda) for a in (x, w, b, off, m, go)]
    out = tx.new_empty(2, 4, 6, 6)
    dcn.modulated_deform_conv_cuda_forward(tx, tw, tb, tx.new_empty(0), toff, tm, out, tx.new_empty(0), 3, 3, 1, 1,
                                           1, 1, 1, 1, 1, 1, True)
    o_ref = capi.dcn_forward(x.astype(np.float64), w.astype(np.float64), b.astype(np.float64), off.astype(np.float64),
                             m.astype(np.float64), 1, 1, 1)
    _close(out.cpu().numpy(), o_ref, "output")
    gw = torch.ones_like(tw)  # accumulation semantics: starts from the caller's values
    gi, gb, goff, gm = torch.zeros_like(tx), torch.zeros_like(tb), torch.zeros_like(toff), torch.zeros_like(tm)
    dcn.modulated_deform_conv_cuda_backward(tx, tw, tb, None, toff, tm, None, gi, gw, gb, goff, gm, tgo, 3, 3, 1, 1,
                                            1, 1, 1, 1, 1, 1, True)
    ref = capi.dcn_backward(x.astype(np.float64), w.astype(np.float64), b.astype(np.float64), off.astype(np.float64),
                            m.astype(np.float64), go.astype(np.float64), 1, 1, 1)
    _close(gw.cpu().numpy(), ref[1] + 1.0, "grad_weight accumulates")
    _close(gb.cpu().numpy(), ref[2], "grad_bias")
    with pytest.raises(RuntimeError, match="contiguous"):
        dcn.modulated_deform_conv_cuda_forward(tx.transpose(2, 3), tw, tb, None, toff, tm, out, None, 3, 3, 1, 1, 1, 1,
                                               1, 1, 1, 1, True)
    with pytest.raises(RuntimeError, match="invalid spatial size of offset"):
        dcn.deform_conv(tx, toff[:, :, :3], tw, 1, 1, 1)


def test_dcn_modules_state_dict_and_zero_init(cuda):
    """ModulatedDeformConvPack: conv_offset_mask zero-init -> offsets 0, mask 0.5: output = 0.5 * plain conv
    (SURVEY.md App. B2.8); parameter names match the reference (modules/deform_conv.py:84-157)."""
    from megreader_b200.dcn import ModulatedDeformConvPack
    torch.manual_seed(0)
    mod = ModulatedDeformConvPack(8, 6, 3, stride=1, padding=1, bias=True).to(cuda)
    assert sorted(mod.state_dict()) == ["bias", "conv_offset_mask.bias", "conv_offset_mask.weight", "weight"]
    x = torch.randn(2, 8, 10, 12, device=cuda)
    ref = 0.5 * torch.nn.functional.conv2d(x, mod.weight, None, 1, 1) + mod.bias.view(1, -1, 1, 1)
    torch.testing.assert_close(mod(x), ref, rtol=1e-4, atol=1e-4)
