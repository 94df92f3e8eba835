"""GPU parity of the CRNN path (SURVEY.md §8 rows A6-A8): megreader_b200's modules behind the reference surfaces vs
golden vectors produced by the UNMODIFIED reference modules on CPU (oracle/make_golden.py crnn; same name-seeded
weights via tests/weights.py), and the 1D CTC head vs the reference's own call (torch CPU ctc_loss in float64,
decoders/crnn.py:47-48,95-99)."""
import os

import numpy as np
import pytest
import torch

from tests.weights import fill_state_dict

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def api():
    import megreader_b200
    megreader_b200.install_reference_api()
    import backbones
    import decoders
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return backbones, decoders


@pytest.mark.parametrize("zero_inf", [True, False])
def test_ctc1d_vs_reference_call(cuda, zero_inf):
    from megreader_b200 import ctc1d
    rng = np.random.RandomState(0)
    T, N, C, S = 26, 7, 38, 32
    logits = torch.from_numpy(rng.standard_normal((T, N, C)).astype(np.float32) * 2)
    lengths = torch.tensor([3, 8, 1, 12, 5, 30, 0])    # 30 labels in T=26 columns: infeasible -> inf / zero_infinity;
    #                                                    0: the blank-only path, nll = -sum_t log p(t, blank) as in torch
    labels = torch.zeros(N, S, dtype=torch.int32)
    for b in range(N):
        labels[b, :lengths[b]] = torch.from_numpy(rng.randint(2, C, size=int(lengths[b])))
    labels[1, 3] = labels[1, 2]                          # repeated label
    ref_in = logits.double().requires_grad_(True)
    ref_lp = torch.nn.functional.log_softmax(ref_in, dim=2)
    ref = torch.nn.CTCLoss(zero_infinity=zero_inf)(ref_lp, labels, torch.full((N,), T, dtype=torch.int32), lengths)
    x = logits.to(cuda).requires_grad_(True)
    loss, lp = ctc1d.ctc_loss_from_logits(x, labels.to(cuda), torch.full((N,), T), lengths.to(cuda), 0, zero_inf, "mean")
    np.testing.assert_allclose(lp.cpu().numpy(), ref_lp.detach().numpy(), rtol=1e-5, atol=1e-5)
    if zero_inf:
        ref.backward()
        np.testing.assert_allclose(loss.item(), ref.item(), rtol=1e-4)
        loss.backward()
        np.testing.assert_allclose(x.grad.cpu().numpy(), ref_in.grad.numpy(), rtol=1e-3, atol=2e-6)
    else:
        assert torch.isinf(ref) and torch.isinf(loss)


@pytest.mark.parametrize("name", ["cfg1", "w128"])
def test_crnn_train_step_vs_reference_golden(cuda, api, name):
    backbones, decoders = api
    g = np.load(os.path.join(GOLD, "crnn_ref_%s.npz" % name))
    bb = fill_state_dict(backbones.crnn_backbone(), "bb.").to(cuda).train()
    dec = fill_state_dict(decoders.CRNNDecoder(in_channels=512, inner_channels=256), "dec.").to(cuda).train()
    x = torch.from_numpy(np.repeat(g["x"], 3, axis=1)).to(cuda)
    feat = bb(x)
    np.testing.assert_allclose(feat.detach().cpu().numpy(), g["feature"], rtol=1e-4, atol=1e-4)
    loss, pred = dec(feat, targets=torch.from_numpy(g["labels"]).to(cuda), lengths=torch.from_numpy(g["lengths"]).to(cuda),
                     train=True)
    assert pred.dtype == torch.float64 and tuple(pred.shape) == g["log_probs"].shape
    np.testing.assert_allclose(pred.cpu().numpy(), g["log_probs"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(loss.item(), float(g["loss"]), rtol=1e-4)
    loss.mean().backward()
    params = dict(list(bb.named_parameters()) + list(dec.named_parameters()))
    for key in g.files:
        if key.startswith("grad."):
            got = params[key[5:]].grad.cpu().numpy()
            scale = max(1e-6, float(np.abs(g[key]).max()))
            np.testing.assert_allclose(got, g[key], rtol=2e-3, atol=max(2e-4 * scale, 1e-6), err_msg=key)  # conv bias before BN: grad == 0 up to noise
        elif key.startswith("gnorm.") and float(g[key]) > 1e-5:   # conv bias before BN: |grad| is noise (~1e-7)
            np.testing.assert_allclose(params[key[6:]].grad.double().norm().item(), float(g[key]), rtol=2e-3, err_msg=key)
        elif key.startswith("bn."):
            np.testing.assert_allclose(bb.state_dict()[key[3:]].cpu().numpy(), g[key], rtol=1e-4, atol=1e-5, err_msg=key)
    # eval branch: softmax (N, C, 1, T); argmax labels must be bit-exact (north_star)
    bb.eval(); dec.eval()
    with torch.no_grad():
        prob = dec(bb(x), train=False)
    assert tuple(prob.shape) == g["eval_prob"].shape
    np.testing.assert_allclose(prob.cpu().numpy(), g["eval_prob"], rtol=1e-3, atol=1e-5)
    assert np.array_equal(prob.argmax(1).cpu().numpy(), g["eval_prob"].argmax(1))


def test_crnn_modules_refuse_cpu(api):
    backbones, decoders = api
    with pytest.raises(NotImplementedError):
        backbones.crnn_backbone()(torch.zeros(1, 3, 32, 32))


def test_ctc_decoder2d_surface(cuda, api):
    """CTCDecoder2D train branch: loss = ctc_loss_2d(log(max(mask*classify, tiny))) / length, pred (T,H,N,C)."""
    from oracle import capi
    _, decoders = api
    torch.manual_seed(0)
    dec = fill_state_dict(decoders.CTCDecoder2D(16, inner_channels=8), "d2.").to(cuda).train()
    feat = torch.randn(3, 16, 4, 10, device=cuda)
    labels = torch.zeros(3, 32, dtype=torch.int32, device=cuda)
    labels[:, :2] = torch.tensor([[5, 9], [7, 7], [30, 2]], device=cuda)
    lengths = torch.tensor([2, 2, 1], device=cuda)
    loss, pred = dec(feat, targets=labels, lengths=lengths, train=True)
    assert tuple(pred.shape) == (10, 4, 3, 38) and tuple(loss.shape) == (3,)
    nll_ref, _ = capi.ctc2d_forward(pred.detach().cpu().numpy().astype(np.float64), labels.cpu().numpy().astype(np.int64),
                                    np.full(3, 10), lengths.cpu().numpy())
    np.testing.assert_allclose(loss.detach().cpu().numpy(), nll_ref / lengths.cpu().numpy(), rtol=1e-4)
    loss.mean().backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in dec.parameters())
    dec.eval()
    classify, mask = dec(feat)
    assert tuple(classify.shape) == (3, 38, 4, 10) and tuple(mask.shape) == (3, 1, 4, 10)


def test_backbone_bn_modes_and_input_gradient(cuda, api):
    """ADVICE r1: BatchNorm's batch-statistics switch follows module.training (also under no_grad), saving for backward
    follows grad mode (also in eval()), and the input gradient is returned when the images require grad.  Reference:
    the same layers as plain torch modules (oracle/crnn_port.py) on the GPU in fp32."""
    from oracle import crnn_port
    backbones, _ = api
    bb = fill_state_dict(backbones.crnn_backbone(), "bb.").to(cuda)
    ref = fill_state_dict(crnn_port.CRNNBackbonePort(), "bb.").to(cuda)
    torch.manual_seed(3)
    x = torch.randn(3, 3, 32, 48, device=cuda)
    # 1) train() under no_grad: batch statistics + running-stat update
    bb.train(); ref.train()
    with torch.no_grad():
        y, yr = bb(x), ref(x)
    torch.testing.assert_close(y, yr, rtol=1e-4, atol=1e-4)
    for k, v in ref.state_dict().items():
        if "running" in k:
            torch.testing.assert_close(bb.state_dict()[k], v, rtol=1e-4, atol=1e-5, msg=k)
    # 2) eval() with grad: running statistics, full backward incl. the input gradient
    bb.eval(); ref.eval()
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    y, yr = bb(xa), ref(xb)
    torch.testing.assert_close(y, yr, rtol=1e-4, atol=1e-4)
    go = torch.randn_like(yr)
    y.backward(go); yr.backward(go)
    torch.testing.assert_close(xa.grad, xb.grad, rtol=1e-3, atol=1e-4 * float(xb.grad.abs().max()))
    for (n, p), (_, q) in zip(bb.named_parameters(), ref.named_parameters()):
        torch.testing.assert_close(p.grad, q.grad, rtol=2e-3, atol=2e-4 * max(1e-6, float(q.grad.abs().max())), msg=n)
    # 3) train() with an input that requires grad; a second backward raises instead of crashing
    bb.train(); ref.train()
    bb.zero_grad(); ref.zero_grad()
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    y, yr = bb(xa), ref(xb)
    y.backward(go, retain_graph=True); yr.backward(go)
    torch.testing.assert_close(xa.grad, xb.grad, rtol=1e-3, atol=1e-4 * float(xb.grad.abs().max()))
    with pytest.raises(RuntimeError, match="retain_graph"):
        y.backward(go)
