"""GPU: fused 2D-CTC head epilogue (csrc/ctc2d_head.cu through the C-ABI) against the reference goldens, against the
CPU oracle on ragged shapes, and the fused logits->loss node against the unfused composition of our own ops."""
import os

import numpy as np
import pytest
import torch
from tests.cases import load_head_golden

from megreader_b200 import ctc2d, ctc2d_head
from oracle import head_port

pytestmark = pytest.mark.gpu


def _close(a, ref, what, tol=2e-5):
    ref = np.asarray(ref)
    scale = max(1.0, float(np.abs(ref).max()))
    np.testing.assert_allclose(a.detach().cpu().numpy(), ref, rtol=tol, atol=tol * scale, err_msg=what)


def _mismatch_fraction(a, ref, tol=1e-4):
    a, ref = a.detach().cpu().numpy(), np.asarray(ref)
    return float((np.abs(a - ref) > tol * (1 + np.abs(ref))).mean())


@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_against_reference_golden(cuda, tag):
    g = load_head_golden()
    m = torch.from_numpy(g[tag + ".mask_logits"]).to(cuda).requires_grad_(True)
    z = torch.from_numpy(g[tag + ".cls_logits"]).to(cuda).requires_grad_(True)
    tiny = float(g[tag + ".tiny"])
    lp = ctc2d_head.head_log_probs(m, z, tiny)
    assert lp.is_contiguous() and tuple(lp.shape) == g[tag + ".pred"].shape
    lp.backward(torch.from_numpy(g[tag + ".grad_pred"]).to(cuda))
    if tag == "b":                       # clamp inactive everywhere: plain closeness
        _close(lp, g[tag + ".pred"], "pred")
        _close(m.grad, g[tag + ".grad_mask_logits"], "d mask logits", 1e-4)
        _close(z.grad, g[tag + ".grad_cls_logits"], "d classify logits", 1e-4)
    else:                                # entries within rounding of the clamp threshold may take the other branch
        assert _mismatch_fraction(lp, g[tag + ".pred"]) == 0.0
        assert _mismatch_fraction(z.grad, g[tag + ".grad_cls_logits"]) < 2e-4
        assert _mismatch_fraction(m.grad, g[tag + ".grad_mask_logits"]) < 2e-3


@pytest.mark.parametrize("shape", [(5, 38, 8, 32), (3, 38, 1, 37), (9, 100, 3, 65), (17, 7, 5, 1), (1, 38, 8, 32),
                                   (3, 64, 4, 40), (2, 41, 3, 33),        # 64-register-row variant of the warp kernels
                                   (2, 2000, 2, 37)])                     # large alphabet: class-tiled kernels
def test_against_oracle_ragged(cuda, shape):
    N, C, H, W = shape
    rng = np.random.RandomState(N * 1000 + C)
    m = torch.from_numpy((rng.standard_normal((N, 1, H, W)) * 2).astype(np.float32))
    z = torch.from_numpy((rng.standard_normal((N, C, H, W)) * 3).astype(np.float32))
    dlp = torch.from_numpy(rng.standard_normal((W, H, N, C)).astype(np.float32))
    ref = head_port.head_log_probs(m.double(), z.double()).float()
    rdm, rdz = head_port.head_grads(m.double(), z.double(), dlp.double())
    mc, zc = m.to(cuda).requires_grad_(True), z.to(cuda).requires_grad_(True)
    lp = ctc2d_head.head_log_probs(mc, zc)
    lp.backward(dlp.to(cuda))
    _close(lp, ref.numpy(), "log_probs")
    _close(zc.grad, rdz.float().numpy(), "d classify logits", 1e-4)
    _close(mc.grad, rdm.float().numpy(), "d mask logits", 1e-4)


def test_fused_loss_equals_composition(cuda):
    """logits -> nll in one node (gradient through the per-(t,class) factor) == head epilogue + ops.ctc_loss_2d."""
    torch.manual_seed(3)
    N, C, H, W, S = 37, 38, 8, 32, 32
    m = (torch.randn(N, 1, H, W, device=cuda) * 2)
    z = (torch.randn(N, C, H, W, device=cuda) * 2)
    lengths = torch.randint(1, 12, (N,), device=cuda)
    targets = torch.zeros(N, S, dtype=torch.long, device=cuda)
    for b in range(N):
        targets[b, :lengths[b]] = torch.randint(2, C, (int(lengths[b]),), device=cuda)
    il = torch.full((N,), W, dtype=torch.long, device=cuda)
    go = torch.rand(N, device=cuda) + 0.5
    m1, z1 = m.clone().requires_grad_(True), z.clone().requires_grad_(True)
    nll1, lp1 = ctc2d_head.head_loss(m1, z1, targets, il, lengths, 0)
    (nll1 * go).sum().backward()
    m2, z2 = m.clone().requires_grad_(True), z.clone().requires_grad_(True)
    lp2 = ctc2d_head.head_log_probs(m2, z2)
    nll2 = ctc2d.ctc_loss_2d(lp2, targets, il, lengths)
    (nll2 * go).sum().backward()
    assert torch.equal(lp1, lp2.detach())
    _close(nll1, nll2.detach().cpu().numpy(), "nll", 1e-6)
    _close(z1.grad, z2.grad.cpu().numpy(), "d classify logits", 2e-5)
    _close(m1.grad, m2.grad.cpu().numpy(), "d mask logits", 2e-5)


def test_large_alphabet_fused_loss(cuda):
    """ChineseCharset-sized head (concern/charsets.py:65-78): logits -> loss through the class-tiled epilogue kernels and the
    CTC factor equals the unfused composition."""
    torch.manual_seed(4)
    N, C, H, W, S = 3, 5000, 2, 12, 8
    m = torch.randn(N, 1, H, W, device=cuda)
    z = torch.randn(N, C, H, W, device=cuda) * 2
    lengths = torch.tensor([3, 5, 1], device=cuda)
    targets = torch.zeros(N, S, dtype=torch.long, device=cuda)
    for b in range(N):
        targets[b, :lengths[b]] = torch.randint(2, C, (int(lengths[b]),), device=cuda)
    il = torch.full((N,), W, dtype=torch.long, device=cuda)
    m1, z1 = m.clone().requires_grad_(True), z.clone().requires_grad_(True)
    nll1, lp1 = ctc2d_head.head_loss(m1, z1, targets, il, lengths, 0)
    nll1.sum().backward()
    m2, z2 = m.clone().requires_grad_(True), z.clone().requires_grad_(True)
    lp2 = ctc2d_head.head_log_probs(m2, z2)
    ref = head_port.head_log_probs(m.cpu().double(), z.cpu().double()).float()
    _close(lp2, ref.numpy(), "log_probs")
    nll2 = ctc2d.ctc_loss_2d(lp2, targets, il, lengths)
    nll2.sum().backward()
    _close(nll1, nll2.detach().cpu().numpy(), "nll", 1e-5)
    _close(z1.grad, z2.grad.cpu().numpy(), "d classify logits", 5e-5)
    _close(m1.grad, m2.grad.cpu().numpy(), "d mask logits", 5e-5)


def test_full_size_normalisation_property(cuda):
    """BASELINE cfg-3 size (N = 2048 samples of 38 x 8 x 32): with the clamp inactive, sum_{h,c} exp(log_probs[t,:,n,:]) == 1
    (softmax over H times softmax over C), and the logits' gradients of any upstream gradient sum to zero over C / over H."""
    torch.manual_seed(5)
    N, C, H, W = 2048, 38, 8, 32
    m = torch.randn(N, 1, H, W, device=cuda).requires_grad_(True)
    z = torch.randn(N, C, H, W, device=cuda).requires_grad_(True)
    lp = ctc2d_head.head_log_probs(m, z)
    total = lp.exp().sum(dim=(1, 3))
    assert float((total - 1).abs().max()) < 1e-4
    lp.backward(torch.randn_like(lp))
    assert float(z.grad.sum(dim=1).abs().max()) < 1e-3 and float(m.grad.sum(dim=2).abs().max()) < 1e-2


def test_refuses_cpu():
    with pytest.raises(NotImplementedError):
        ctc2d_head.head_log_probs(torch.zeros(1, 1, 2, 2), torch.zeros(1, 3, 2, 2))
