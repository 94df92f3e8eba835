"""GPU: every building block of the CRNN engine (csrc/nn_kernels.cu, csrc/gemm.cu) against the plain PyTorch fp32
reference of the same op (the ATen ops the reference's modules call), fp32 mode tight, bf16 mode loose."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops(cuda):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from megreader_b200 import nnops
    return nnops


def _tol(dtype):
    return dict(rtol=1e-5, atol=1e-5) if dtype == torch.float32 else dict(rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("geo", [(2, 6, 9, 8, 3, 3, 1, 1), (3, 2, 7, 16, 2, 2, 0, 0), (1, 5, 4, 8, 3, 3, 1, 1)])
def test_im2col_col2im(cuda, ops, dtype, geo):
    N, H, W, C, kh, kw, ph, pw = geo
    torch.manual_seed(0)
    x = torch.randn(N, H, W, C, device=cuda).to(dtype)
    K = kh * kw * C
    col, Ho, Wo = ops.im2col(x, kh, kw, ph, pw, K)
    ref = F.unfold(x.float().permute(0, 3, 1, 2), (kh, kw), padding=(ph, pw))        # [N, C*kh*kw, L], row = c*kh*kw + tap
    ref = ref.view(N, C, kh * kw, Ho * Wo).permute(0, 3, 2, 1).reshape(N * Ho * Wo, K)
    torch.testing.assert_close(col.float(), ref, rtol=0, atol=0)
    d = torch.randn(N * Ho * Wo, K, device=cuda).to(dtype)
    dx = ops.col2im(d, N, H, W, C, kh, kw, ph, pw)
    refd = d.float().view(N, Ho * Wo, kh * kw, C).permute(0, 3, 2, 1).reshape(N, C * kh * kw, Ho * Wo)
    refx = F.fold(refd, (H, W), (kh, kw), padding=(ph, pw)).permute(0, 2, 3, 1)
    torch.testing.assert_close(dx.float(), refx, **_tol(dtype))


def test_im2col_padded_k_and_layout_conversion(cuda, ops):
    x = torch.randn(2, 3, 6, 10, device=cuda)
    a = ops.nchw_to_nhwc(x, 4, torch.float32)
    assert torch.equal(a[..., :3], x.permute(0, 2, 3, 1)) and torch.all(a[..., 3] == 0)
    col, Ho, Wo = ops.im2col(a, 3, 3, 1, 1, 40)
    assert col.shape == (2 * 6 * 10, 40) and torch.all(col[:, 36:] == 0)
    back = ops.nhwc_to_nchw(a, 3)
    assert torch.equal(back, x)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("pool", [((2, 2), (2, 2), (0, 0)), ((2, 2), (2, 1), (0, 1))])
def test_bias_relu_pool(cuda, ops, dtype, pool):
    k, s, p = pool
    N, H, W, C = 3, 8, 10, 16
    torch.manual_seed(1)
    z = torch.randn(N * H * W, C, device=cuda).to(dtype)
    bias = torch.randn(C, device=cuda)
    y, idx = ops.bias_relu_pool_fwd(z, bias, N, H, W, C, k, s, p)
    zr = z.float().view(N, H, W, C).permute(0, 3, 1, 2).requires_grad_(True)
    act = F.relu(zr + bias.view(1, -1, 1, 1)).to(dtype).float()
    ref = F.max_pool2d(act, k, s, p)
    torch.testing.assert_close(y.float().permute(0, 3, 1, 2), ref, rtol=0, atol=0)
    dy = torch.randn_like(ref).to(dtype)
    ref.backward(dy.float())
    dz, dbias = ops.bias_relu_pool_bwd(dy.permute(0, 2, 3, 1).contiguous(), y, idx, N, H, W, C, k, s, p)
    torch.testing.assert_close(dz.float().view(N, H, W, C).permute(0, 3, 1, 2), zr.grad, **_tol(dtype))
    torch.testing.assert_close(dbias, dz.float().sum(0), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_batchnorm_train(cuda, ops, dtype):
    rows, C = 3000, 32
    torch.manual_seed(2)
    z = (torch.randn(rows, C, device=cuda) * 2 + 0.5).to(dtype)
    bias = torch.randn(C, device=cuda)
    gamma = torch.rand(C, device=cuda) + 0.5
    beta = torch.randn(C, device=cuda)
    rm, rv = torch.zeros(C, device=cuda), torch.ones(C, device=cuda)
    rm_ref, rv_ref = rm.clone(), rv.clone()
    y, mean, invstd = ops.bn_train_fwd(z, bias, gamma, beta, rm, rv, 0.1, 1e-5)
    zr = z.float().requires_grad_(True)
    ref = F.batch_norm((zr + bias).t().reshape(1, C, rows), rm_ref, rv_ref, gamma, beta, True, 0.1, 1e-5)
    ref = ref.reshape(C, rows).t()
    torch.testing.assert_close(y.float(), ref, **_tol(dtype))
    torch.testing.assert_close(rm, rm_ref, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(rv, rv_ref, rtol=1e-4, atol=1e-5)
    dy = torch.randn(rows, C, device=cuda).to(dtype)
    g = torch.autograd.grad(ref, zr, dy.float())[0]
    dx, dgamma, dbeta, dbias = ops.bn_train_bwd(dy, z, bias, mean, invstd, gamma)
    torch.testing.assert_close(dbias, dx.float().sum(0), rtol=1e-3, atol=2e-2)
    torch.testing.assert_close(dx.float(), g, rtol=1e-3, atol=1e-4 if dtype == torch.float32 else 3e-2)
    xhat = (z.float() + bias - mean) * invstd
    torch.testing.assert_close(dbeta, dy.float().sum(0), rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(dgamma, (dy.float() * xhat).sum(0), rtol=1e-3, atol=1e-2)
    torch.testing.assert_close(ops.colsum(dy), dy.float().sum(0), rtol=1e-4, atol=1e-3)
    odd = torch.randn(500, 38, device=cuda)
    torch.testing.assert_close(ops.colsum(odd), odd.sum(0), rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(ops.bias_act(odd, torch.arange(38., device=cuda), relu=True),
                               F.relu(odd + torch.arange(38., device=cuda)))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_gemm_variants(cuda, ops, dtype):
    torch.manual_seed(3)
    M, N, K = 70, 50, 96
    A, B = torch.randn(M, K, device=cuda).to(dtype), torch.randn(K, N, device=cuda).to(dtype)
    ref = A.float() @ B.float()
    tol = dict(rtol=1e-4, atol=1e-4) if dtype == torch.float32 else dict(rtol=2e-2, atol=0.3)
    torch.testing.assert_close(ops.gemm(A, B).float(), ref, **tol)
    torch.testing.assert_close(ops.gemm(A, B.t().contiguous(), transB=True).float(), ref, **tol)
    torch.testing.assert_close(ops.gemm(A.t().contiguous(), B, transA=True, out_dtype=torch.float32), ref,
                               **(tol if dtype == torch.float32 else dict(rtol=1e-3, atol=1e-3)))
    out = torch.ones(M, N, device=cuda)
    ops.gemm(A, B, out=out, beta=1.0)
    torch.testing.assert_close(out, ref + 1, **(tol if dtype == torch.float32 else dict(rtol=1e-3, atol=1e-3)))
    wide = torch.randn(M, 2 * K, device=cuda).to(dtype)
    torch.testing.assert_close(ops.gemm(wide[:, K:], B, out_dtype=torch.float32), wide[:, K:].float() @ B.float(),
                               **(tol if dtype == torch.float32 else dict(rtol=1e-3, atol=1e-3)))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_bilstm_layer_vs_torch(cuda, dtype):
    """BidirectionalLSTM (decoders/crnn.py:8-24) forward + all gradients vs nn.LSTM + nn.Linear in fp32."""
    from megreader_b200 import crnn_engine
    torch.manual_seed(4)
    T, N, I, H, O = 7, 5, 16, 8, 24
    rnn = torch.nn.LSTM(I, H, bidirectional=True).to(cuda)
    emb = torch.nn.Linear(2 * H, O).to(cuda)

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.rnn, self.embedding = rnn, emb
    m = M()
    x = torch.randn(T, N, I, device=cuda)
    xr = x.clone().requires_grad_(True)
    rec, _ = rnn(xr)
    ref = emb(rec.view(T * N, 2 * H)).view(T, N, O)
    dout = torch.randn_like(ref)
    ref.backward(dout)
    ref_grads = [p.grad.clone() for p in crnn_engine._bilstm_params(m)]
    for p in m.parameters():
        p.grad = None
    crnn_engine.set_compute_dtype(dtype)
    try:
        xe = x.clone().requires_grad_(True)
        out = crnn_engine.bilstm_forward(m, xe)
        out.float().backward(dout)
    finally:
        crnn_engine.set_compute_dtype(torch.float32)
    tol = dict(rtol=1e-3, atol=3e-4) if dtype == torch.float32 else dict(rtol=5e-2, atol=5e-2)
    torch.testing.assert_close(out.float(), ref, **tol)
    torch.testing.assert_close(xe.grad, xr.grad, **tol)
    for got, want in zip([p.grad for p in crnn_engine._bilstm_params(m)], ref_grads):
        torch.testing.assert_close(got, want, **(tol if dtype == torch.float32 else dict(rtol=5e-2, atol=0.15)))


def _bilstm_case(cuda, T, N, I, H, O, seed):
    from megreader_b200 import crnn_engine
    torch.manual_seed(seed)
    rnn = torch.nn.LSTM(I, H, bidirectional=True).to(cuda)
    emb = torch.nn.Linear(2 * H, O).to(cuda)

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.rnn, self.embedding = rnn, emb
    m = M()
    x = torch.randn(T, N, I, device=cuda)
    xr = x.clone().requires_grad_(True)
    rec, _ = rnn(xr)
    ref = emb(rec.view(T * N, 2 * H)).view(T, N, O)
    dout = torch.randn_like(ref)
    ref.backward(dout)
    ref_grads = [p.grad.clone() for p in crnn_engine._bilstm_params(m)]
    return m, x, dout, ref, xr.grad, ref_grads


def _bilstm_run(m, x, dout, mode):
    from megreader_b200 import crnn_engine
    for p in m.parameters():
        p.grad = None
    crnn_engine.set_compute_dtype(torch.bfloat16)
    before = crnn_engine.LSTM_MODE
    crnn_engine.LSTM_MODE = mode
    try:
        xe = x.clone().requires_grad_(True)
        out = crnn_engine.bilstm_forward(m, xe)
        out.float().backward(dout)
        torch.cuda.synchronize()
    finally:
        crnn_engine.set_compute_dtype(torch.float32)
        crnn_engine.LSTM_MODE = before
    return out.float(), xe.grad, [p.grad.clone() for p in crnn_engine._bilstm_params(m)]


@pytest.mark.parametrize("mode", ["step", "seq"])
@pytest.mark.parametrize("shape", [(6, 150, 64, 64, 40), (9, 512, 128, 256, 38), (1, 7, 64, 64, 8)])
def test_bilstm_fused_tcgen05_paths(cuda, mode, shape):
    """H % 64 == 0 in bf16 mode: per-step fused wgmma kernels ("step") and the persistent whole-sequence kernels
    ("seq", csrc/lstm_seq_tcgen05.cu) against nn.LSTM + nn.Linear in fp32."""
    from megreader_b200 import crnn_engine
    m, x, dout, ref, ref_dx, ref_grads = _bilstm_case(cuda, *shape, seed=6)
    out, dx, grads = _bilstm_run(m, x, dout, mode)
    if mode == "seq":
        assert int(crnn_engine.LAST_LSTM_FLAGS[-1]) == 0, "inter-CTA wait timed out"
    torch.testing.assert_close(out, ref, rtol=5e-2, atol=5e-2)
    torch.testing.assert_close(dx, ref_dx, rtol=5e-2, atol=0.02 * float(ref_dx.abs().max()) + 5e-2)
    for got, want in zip(grads, ref_grads):
        torch.testing.assert_close(got, want, rtol=5e-2, atol=0.02 * float(want.abs().max()) + 0.05)


@pytest.mark.parametrize("shape", [(26, 300, 512, 256, 256), (65, 512, 256, 256, 38), (5, 1100, 64, 128, 16)])
def test_bilstm_persistent_equals_stepwise(cuda, shape):
    """The persistent kernels run the same arithmetic as the per-step fused kernels (same tiles, same accumulation
    order), at the CRNN shapes (T = 26 / 65, N = 512, H = 256), with a ragged last row tile and with > 8 row tiles:
    outputs and every gradient agree to bf16 rounding of the last step."""
    from megreader_b200 import crnn_engine
    m, x, dout, _, _, _ = _bilstm_case(cuda, *shape, seed=8)
    out_a, dx_a, g_a = _bilstm_run(m, x, dout, "step")
    out_b, dx_b, g_b = _bilstm_run(m, x, dout, "seq")
    assert int(crnn_engine.LAST_LSTM_FLAGS[-1]) == 0, "inter-CTA wait timed out"
    torch.testing.assert_close(out_b, out_a, rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(dx_b, dx_a, rtol=1e-2, atol=1e-2 * float(dx_a.abs().max()) + 1e-3)
    for got, want in zip(g_b, g_a):
        torch.testing.assert_close(got, want, rtol=1e-2, atol=1e-2 * float(want.abs().max()) + 1e-3)


def test_adam_matches_torch(cuda, ops):
    torch.manual_seed(5)
    p = torch.randn(1000, device=cuda)
    ref = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=1e-3)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    shadow = torch.empty(1000, dtype=torch.bfloat16, device=cuda)
    for step in range(1, 4):
        g = torch.randn(1000, device=cuda)
        ref.grad = g.clone()
        opt.step()
        ops.adam_step(p, g, m, v, 1e-3, 0.9, 0.999, 1e-8, step, 1.0, shadow)
    torch.testing.assert_close(p, ref.detach(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(shadow.float(), p, rtol=1e-2, atol=1e-2)


def test_crnn_bf16_mode_close_to_fp32_golden(cuda):
    """bf16 compute (BASELINE.json cfg 2) vs the reference's fp32 golden: reported as a delta, loose bound."""
    import os
    import megreader_b200
    from megreader_b200 import crnn_engine
    from tests.weights import fill_state_dict
    megreader_b200.install_reference_api()
    import backbones
    import decoders
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "crnn_ref_cfg1.npz"))
    bb = fill_state_dict(backbones.crnn_backbone(), "bb.").to(cuda).train()
    dec = fill_state_dict(decoders.CRNNDecoder(in_channels=512, inner_channels=256), "dec.").to(cuda).train()
    crnn_engine.set_compute_dtype(torch.bfloat16)
    try:
        x = torch.from_numpy(np.repeat(g["x"], 3, axis=1)).to(cuda)
        loss, pred = dec(bb(x), targets=torch.from_numpy(g["labels"]).to(cuda),
                         lengths=torch.from_numpy(g["lengths"]).to(cuda), train=True)
        loss.mean().backward()
    finally:
        crnn_engine.set_compute_dtype(torch.float32)
    assert abs(loss.item() - float(g["loss"])) / float(g["loss"]) < 3e-2
    gn = dec.rnn[1].embedding.weight.grad.double().norm().item()
    assert abs(gn - float(g["gnorm.rnn.1.embedding.weight"])) / float(g["gnorm.rnn.1.embedding.weight"]) < 0.1


def test_weight_pack_kernels(cuda, ops):
    """one-launch weight layout packs == the permute / pad / flip / gather / cast chains they replace (bit-exact)."""
    torch.manual_seed(9)
    for (Cout, Cin, kh, kw, Cp) in [(64, 3, 3, 3, 8), (128, 64, 3, 3, 64), (512, 512, 2, 2, 512)]:
        w = torch.randn(Cout, Cin, kh, kw, device=cuda)
        K = kh * kw * Cp
        Kp = -(-K // 8) * 8 + 8
        ref = torch.nn.functional.pad(w.permute(0, 2, 3, 1), (0, Cp - Cin)).reshape(Cout, K)
        ref = torch.nn.functional.pad(ref, (0, Kp - K)).bfloat16()
        assert torch.equal(ops.conv_weight_pack(w, Cp, Kp, torch.bfloat16, 0), ref)
        if Cp == Cin:
            refd = w.flip(2, 3).permute(1, 2, 3, 0).reshape(Cin, kh * kw * Cout).contiguous()
            assert torch.equal(ops.conv_weight_pack(w, Cp, K, torch.float32, 1), refd)
    H = 64
    perm = torch.arange(4 * H, device=cuda).view(4, H).t().reshape(-1)
    a, b = torch.randn(4 * H, 96, device=cuda), torch.randn(4 * H, 96, device=cuda)
    assert torch.equal(ops.gate_rows_permute(a, H, torch.bfloat16), a[perm].bfloat16())
    assert torch.equal(ops.gate_rows_permute(a[:, 0].contiguous(), H, torch.float32, b=b[:, 0].contiguous()), (a[:, 0] + b[:, 0])[perm])
    um = ops.gate_rows_permute(a, H, torch.float32)
    assert torch.equal(ops.gate_rows_permute(um, H, torch.float32, inverse=True), a)
