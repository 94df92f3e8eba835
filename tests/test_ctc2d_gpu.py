"""GPU parity: the sm_90a 2D-CTC kernels (through the C-ABI) against the CPU oracle on the same seeded
inputs, against the committed golden vectors, and through size-independent properties at full size."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import capi
from tests.cases import ctc2d_case

pytestmark = pytest.mark.gpu

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ctc2d_pyref_*.npz")))
RTOL = 1e-4  # north_star: fp32 loss within 1e-4 relative


def _dev(cuda, *arrs):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(cuda) for a in arrs]


def _oracle(lp, tg, il, tl, go):
    lp64 = lp.astype(np.float64)
    nll, la = capi.ctc2d_forward(lp64, tg, il, tl)
    gr = capi.ctc2d_backward(go.astype(np.float64), lp64, tg, il, tl, nll, la)
    return nll, la, gr


def _check_alpha(la_gpu, la_ref):
    la_gpu = la_gpu.cpu().numpy()
    fin = np.isfinite(la_ref)
    assert np.array_equal(np.isfinite(la_gpu), fin), "log_alpha -inf pattern differs"
    assert np.all(la_gpu[~fin] == la_ref[~fin])
    np.testing.assert_allclose(la_gpu[fin], la_ref[fin], rtol=RTOL, atol=1e-4)


CASES = [
    # seed, T, H, N, C, S, Lmax, ragged
    (1, 32, 8, 32, 38, 32, 12, False),   # cfg-3 per-GPU shape (SURVEY.md §8)
    (2, 32, 8, 7, 38, 32, 12, True),     # ragged input lengths, N not a multiple of the CTA group
    (3, 8, 4, 4, 6, 5, 3, False),
    (4, 12, 1, 3, 7, 6, 4, True),        # H = 1
    (5, 16, 3, 5, 5, 8, 6, False),       # tiny alphabet -> repeated labels
    (6, 20, 2, 9, 11, 40, 9, True),      # 2S+1 = 81 states
    (7, 6, 5, 3, 4001, 3, 3, False),     # large alphabet (falls off the staged path)
    (8, 40, 9, 6, 13, 2, 2, False),      # H > 8
]


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("case", CASES, ids=[str(c[0]) for c in CASES])
def test_contract_forward_backward_vs_oracle(cuda, case, fast, monkeypatch):
    from megreader_b200 import ctc2d
    monkeypatch.setattr(ctc2d, "FAST_MATH", fast)
    seed, T, H, N, C, S, Lmax, ragged = case
    lp, tg, il, tl = ctc2d_case(seed, T, H, N, C, S, Lmax, ragged_T=ragged)
    go = (1.0 / tl).astype(np.float32)
    nll_ref, la_ref, gr_ref = _oracle(lp, tg, il, tl, go)
    d_lp, d_tg, d_il, d_tl, d_go = _dev(cuda, lp, tg, il, tl, go)
    nll, la = ctc2d.ctc2d_forward(d_lp, d_tg, d_il, d_tl, 0, 0.0)
    assert la.shape == (N, T, H, 2 * S + 1) and nll.shape == (N,)
    np.testing.assert_allclose(nll.cpu().numpy(), nll_ref, rtol=RTOL)
    _check_alpha(la, la_ref)
    gr = ctc2d.ctc2d_backward(d_go, d_lp, d_tg, d_il, d_tl, nll, la, 0)
    g = gr.cpu().numpy()
    assert np.array_equal(g == 0, gr_ref == 0), "zero pattern of the gradient differs (K3 :506-513)"
    np.testing.assert_allclose(g, gr_ref, rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize("case", CASES[:6], ids=[str(c[0]) for c in CASES[:6]])
def test_training_pair_equals_contract_path(cuda, case):
    from megreader_b200 import ctc2d
    seed, T, H, N, C, S, Lmax, ragged = case
    lp, tg, il, tl = ctc2d_case(seed, T, H, N, C, S, Lmax, ragged_T=ragged)
    go = (1.0 / tl).astype(np.float32)
    nll_ref, _, gr_ref = _oracle(lp, tg, il, tl, go)
    d_lp, d_tg, d_il, d_tl, d_go = _dev(cuda, lp, tg, il, tl, go)
    d_lp.requires_grad_(True)
    loss = ctc2d.ctc_loss_2d(d_lp, d_tg, d_il, d_tl)
    np.testing.assert_allclose(loss.detach().cpu().numpy(), nll_ref, rtol=RTOL)
    (loss * d_go).sum().backward()
    g = d_lp.grad.cpu().numpy()
    assert np.array_equal(g == 0, gr_ref == 0)
    np.testing.assert_allclose(g, gr_ref, rtol=2e-4, atol=2e-5)


def test_float64_kernels(cuda):
    from megreader_b200 import ctc2d
    lp, tg, il, tl = ctc2d_case(21, 16, 4, 6, 10, 8, 6, ragged_T=True, dtype=np.float64)
    go = np.ones(6)
    nll_ref, la_ref, gr_ref = _oracle(lp, tg, il, tl, go)
    d_lp, d_tg, d_il, d_tl, d_go = _dev(cuda, lp, tg, il, tl, go)
    nll, la = ctc2d.ctc2d_forward(d_lp, d_tg, d_il, d_tl, 0, 0.0)
    np.testing.assert_allclose(nll.cpu().numpy(), nll_ref, rtol=1e-10)
    fin = np.isfinite(la_ref)
    np.testing.assert_allclose(la.cpu().numpy()[fin], la_ref[fin], rtol=1e-9, atol=1e-9)
    gr = ctc2d.ctc2d_backward(d_go, d_lp, d_tg, d_il, d_tl, nll, la, 0)
    np.testing.assert_allclose(gr.cpu().numpy(), gr_ref, rtol=1e-8, atol=1e-10)


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_golden_reference_python(cuda, path):
    """nll vs the reference's python CTCLoss2D; gradient vs its autograd (+exp(lp) on non-zero entries)."""
    from megreader_b200 import ctc2d
    d = np.load(path)
    d_lp, d_tg, d_il, d_tl = _dev(cuda, d["log_probs"], d["targets"], d["input_lengths"], d["target_lengths"])
    nll, la = ctc2d.ctc2d_forward(d_lp, d_tg, d_il, d_tl, 0, 0.0)
    np.testing.assert_allclose(nll.cpu().numpy(), d["ref_nll"], rtol=RTOL)
    g = ctc2d.ctc2d_backward(torch.ones_like(nll), d_lp, d_tg, d_il, d_tl, nll, la, 0).cpu().numpy()
    true_grad = np.where(g != 0, g - np.exp(d["log_probs"].astype(np.float64)), 0.0)
    np.testing.assert_allclose(true_grad, d["ref_autograd"], atol=2e-5)


def test_module_surface_and_reduction(cuda):
    from megreader_b200.ctc2d import CTC2DLoss, CTCLoss2D
    assert CTC2DLoss is CTCLoss2D
    d = np.load(GOLD[0])
    lp = torch.from_numpy(d["log_probs"]).to(cuda)
    # split lp into (mask, classify) any way that sums back
    mask = lp.logsumexp(3)
    classify = lp - mask.unsqueeze(-1)
    tl = torch.from_numpy(d["target_lengths"])
    out = CTCLoss2D(reduction="mean")(mask, classify, torch.from_numpy(d["targets"]),
                                      torch.from_numpy(d["input_lengths"]), tl)
    np.testing.assert_allclose(out.cpu().numpy(), d["ref_nll"] / d["target_lengths"], rtol=RTOL)


def test_errors_match_reference(cuda):
    from megreader_b200 import ctc2d
    lp, tg, il, tl = ctc2d_case(1, 8, 2, 3, 5, 4)
    d_lp, d_tg, d_il, d_tl = _dev(cuda, lp, tg, il, tl)
    with pytest.raises(RuntimeError, match="contiguous"):
        ctc2d.ctc2d_forward(d_lp.permute(1, 0, 2, 3), d_tg, d_il, d_tl, 0, 0.0)
    with pytest.raises(RuntimeError, match="blank must be in label range"):
        ctc2d.ctc2d_forward(d_lp, d_tg, d_il, d_tl, 5, 0.0)
    with pytest.raises(RuntimeError, match="input_lengths must be of size batch_size"):
        ctc2d.ctc2d_forward(d_lp, d_tg, d_il[:2], d_tl, 0, 0.0)
    with pytest.raises(RuntimeError, match="max target length out of range"):
        ctc2d.ctc2d_forward(d_lp, torch.zeros(3, 600, dtype=torch.long, device=cuda), d_il, d_tl, 0, 0.0)
    with pytest.raises(NotImplementedError):
        ctc2d.ctc_loss_2d(torch.from_numpy(lp), torch.from_numpy(tg), torch.from_numpy(il), torch.from_numpy(tl))
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        ctc2d.ctc2d_forward(torch.from_numpy(lp), d_tg, d_il, d_tl, 0, 0.0)


def test_strided_targets_and_empty_batch(cuda):
    from megreader_b200 import ctc2d
    lp, tg, il, tl = ctc2d_case(9, 10, 3, 4, 7, 5, 4)
    d_lp, d_tg, d_il, d_tl = _dev(cuda, lp, tg, il, tl)
    wide = torch.zeros(4, 10, dtype=torch.long, device=cuda)
    wide[:, ::2] = d_tg
    nll_a, _ = ctc2d.ctc2d_forward(d_lp, d_tg, d_il, d_tl, 0, 0.0)
    nll_b, _ = ctc2d.ctc2d_forward(d_lp, wide[:, ::2], d_il, d_tl, 0, 0.0)   # kernel.cu:246 honours target strides
    assert torch.equal(nll_a, nll_b)
    e = ctc2d.ctc2d_forward(torch.empty(10, 3, 0, 7, device=cuda), torch.empty(0, 5, dtype=torch.long, device=cuda),
                            torch.empty(0, dtype=torch.long, device=cuda), torch.empty(0, dtype=torch.long, device=cuda), 0, 0.0)
    assert e[0].numel() == 0 and e[1].shape == (0, 10, 3, 11)


def test_full_size_properties(cuda):
    """cfg-3 shape at a saturating batch (N=4096): properties that need no oracle.
    (1) H-replication: duplicating every height row adds log(2) per column to the likelihood;
    (2) the per-column posterior mass: sum_c exp(Q)*(...)  => sum over (h,c in target) of -true_grad == 1 per t<Tb;
    (3) permuting the batch permutes the outputs bit-exactly."""
    from megreader_b200 import ctc2d
    T, H, N, C, S = 32, 8, 4096, 38, 32
    lp, tg, il, tl = ctc2d_case(3, T, H, N, C, S, 12)
    d_lp, d_tg, d_il, d_tl = _dev(cuda, lp, tg, il, tl)
    nll, la = ctc2d.ctc2d_forward(d_lp, d_tg, d_il, d_tl, 0, 0.0)
    assert torch.isfinite(nll).all()
    # (3)
    perm = torch.randperm(N, device=cuda, generator=torch.Generator(device=cuda).manual_seed(0))
    nll_p, _ = ctc2d.ctc2d_forward(d_lp[:, :, perm].contiguous(), d_tg[perm], d_il[perm], d_tl[perm], 0, 0.0)
    assert torch.equal(nll_p, nll[perm])
    # (1)
    lp2 = torch.cat([d_lp, d_lp], dim=1).contiguous()
    nll2, _ = ctc2d.ctc2d_forward(lp2, d_tg, d_il, d_tl, 0, 0.0)
    np.testing.assert_allclose((nll - nll2).cpu().numpy(), T * np.log(2.0), rtol=1e-4)
    # (2)  -true_grad = exp(G + nll - lp) = posterior of passing (t,h,c); summed over h,c it is 1
    g = ctc2d.ctc2d_backward(torch.ones_like(nll), d_lp, d_tg, d_il, d_tl, nll, la, 0)
    post = torch.where(g != 0, d_lp.exp() - g, torch.zeros_like(g)).sum(dim=(1, 3))  # [T,N]
    np.testing.assert_allclose(post.cpu().numpy(), 1.0, rtol=0, atol=2e-3)
    # oracle spot check on the first 16 samples
    sl = slice(0, 16)
    nll_ref, la_ref, _ = _oracle(lp[:, :, sl], tg[sl], il[sl], tl[sl], np.ones(16))
    np.testing.assert_allclose(nll[sl].cpu().numpy(), nll_ref, rtol=RTOL)
    _check_alpha(la[sl], la_ref)
