"""The fused CRNN stem (csrc/crnn_stem.cu: layer 0 = Conv2d(3, 64, 3, 1, 1) -> ReLU -> MaxPool2d(2, 2)) against a float64
restatement with the same bf16 roundings, against the unfused im2col + GEMM + pool route it replaces, under CUDA-graph
replay, and inside the engine's bf16 training step.  The refusals need no GPU."""
import pytest
import torch
import torch.nn.functional as F

from megreader_b200 import _lib

SHAPES = [(3, 32, 48), (4, 32, 100), (2, 32, 101), (512, 32, 256)]
POOL = torch.nn.MaxPool2d(2, 2)


def _conv(seed, dev):
    torch.manual_seed(seed)
    return torch.nn.Conv2d(3, 64, 3, 1, 1).to(dev)


def _inputs(seed, n, h, w, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn((n, 3, h, w), generator=g, device=dev)
    dy = torch.randn((n, h // 2, w // 2, 64), generator=g, device=dev).to(torch.bfloat16)
    return x, dy


def _bf(t):
    return t.to(torch.bfloat16).double()


def _ulp(v):
    """one bf16 ulp at |v| (8 significant bits)"""
    return torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -120))) - 7)


def _windows(t):
    """[N, C, H, W] -> [N, H/2, W/2, C, 4] with the 2x2 windows in (i, j) order (floor mode: an odd last row / column drops)"""
    n, c, h, w = t.shape
    t = t[:, :, :h // 2 * 2, :w // 2 * 2].reshape(n, c, h // 2, 2, w // 2, 2)
    return t.permute(0, 2, 4, 1, 3, 5).reshape(n, h // 2, w // 2, c, 4)


def _reference_fwd(x, conv):
    """float64 conv of the bf16-rounded operands, then the unfused path's two roundings and the pool"""
    z64 = F.conv2d(_bf(x), _bf(conv.weight.detach()), padding=1)
    z = z64.to(torch.bfloat16).float()
    a = (z + conv.bias.detach().float()[None, :, None, None]).clamp_min(0).to(torch.bfloat16).double()
    win = _windows(a)
    pre64 = _windows((z64 + conv.bias.detach().double()[None, :, None, None]).clamp_min(0))
    return win.max(-1).values, win.argmax(-1), pre64, _windows(z64.abs()).max(-1).values


def _old_route(x, conv):
    """layer 0 as the engine runs it without the stem: NCHW -> NHWC (C padded to 8), im2col, GEMM, bias + ReLU + pool"""
    from megreader_b200 import nnops as ops
    n, _, h, w = x.shape
    a = ops.nchw_to_nhwc(x.contiguous(), 8, torch.bfloat16)
    col, ho, wo = ops.im2col(a, 3, 3, 1, 1, 72)
    Wm = ops.conv_weight_pack(conv.weight, 8, 72, torch.bfloat16, 0)
    z = ops.gemm(col, Wm, transB=True)
    y, idx = ops.bias_relu_pool_fwd(z, conv.bias.detach(), n, ho, wo, 64, (2, 2), (2, 2), (0, 0))
    return y, idx, z, col


def _check_fwd(y, idx, y_ref, arg_ref, pre64, zmax):
    y = y.double()
    tol = _ulp(torch.maximum(y_ref.abs(), zmax))
    assert bool(((y - y_ref).abs() <= tol).all()), float(((y - y_ref).abs() / tol).max())
    top2 = pre64.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > 2 * _ulp(top2[..., 0])
    pos = y > 0
    assert bool((idx[pos & clear] == arg_ref[pos & clear]).all())
    assert bool((idx[~pos] == 4).all()) and bool((idx[pos] < 4).all())      # routing byte 4: pooled value not > 0


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_forward_vs_float64_and_old_route(cuda, shape):
    from megreader_b200 import nnops as ops
    n, h, w = shape
    conv = _conv(1, cuda)
    x, _ = _inputs(2, n, h, w, cuda)
    y, idx = ops.crnn_stem_fwd(x, conv, POOL, True)
    assert y.shape == (n, h // 2, w // 2, 64) and y.dtype == torch.bfloat16 and idx.shape == y.shape
    y_ref, arg_ref, pre64, zmax = _reference_fwd(x, conv)
    _check_fwd(y, idx, y_ref, arg_ref, pre64, zmax)
    y_old, idx_old, _, _ = _old_route(x, conv)
    _check_fwd(y, idx, y_old.double(), idx_old.long(), pre64, zmax)


def _reference_bwd(x, dy, idx):
    """dW [64, 3, 3, 3] and dbias in float64 from the routing: dz = dy where the byte names the window position, else 0"""
    n, hp, wp, c = dy.shape
    sel = idx.long()[..., None] == torch.arange(4, device=dy.device)
    dz = (dy.double()[..., None] * sel).reshape(n, hp, wp, c, 2, 2).permute(0, 3, 1, 4, 2, 5).reshape(n, c, 2 * hp, 2 * wp)
    dz = F.pad(dz, (0, x.shape[3] - 2 * wp, 0, x.shape[2] - 2 * hp))
    dw = torch.nn.grad.conv2d_weight(_bf(x), (64, 3, 3, 3), dz, padding=1)
    return dw, dz.sum((0, 2, 3))


def _rel(a, b):
    return float((a.double() - b).norm() / b.norm())


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_backward_vs_float64_and_repeatable(cuda, shape):
    from megreader_b200 import nnops as ops
    n, h, w = shape
    conv = _conv(3, cuda)
    x, dy = _inputs(4, n, h, w, cuda)
    _, idx = ops.crnn_stem_fwd(x, conv, POOL, True)
    dw, db = ops.crnn_stem_bwd(x, dy, idx, conv, POOL)
    dw_ref, db_ref = _reference_bwd(x, dy, idx)
    assert dw.shape == (64, 3, 3, 3) and db.shape == (64,)
    assert _rel(dw, dw_ref) <= 1e-5 and _rel(db, db_ref) <= 1e-5, (_rel(dw, dw_ref), _rel(db, db_ref))
    dw2, db2 = ops.crnn_stem_bwd(x, dy, idx, conv, POOL)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)


@pytest.mark.gpu
def test_nan_weight_propagates_like_aten(cuda):
    """One NaN weight makes its output channel NaN before the ReLU.  ATen's relu and max_pool2d keep the NaN, so the pooled
    channel is NaN (not 0) and routes no gradient (threshold_backward); every other channel is unchanged."""
    from megreader_b200 import nnops as ops
    n, h, w = 3, 32, 48
    conv = _conv(11, cuda)
    co = 17
    with torch.no_grad():
        conv.weight[co, 1, 2, 0] = float("nan")
    x, dy = _inputs(12, n, h, w, cuda)
    y, idx = ops.crnn_stem_fwd(x, conv, POOL, True)
    assert bool(torch.isnan(y[..., co]).all()), "a NaN pre-activation must survive ReLU + max-pool"
    assert bool((idx[..., co] == 4).all())
    want = F.max_pool2d(F.relu(F.conv2d(x, conv.weight, conv.bias, padding=1)), 2, 2)
    assert bool(torch.isnan(want[:, co]).all())
    keep = torch.arange(64, device=cuda) != co
    y_ref, arg_ref, pre64, zmax = _reference_fwd(x, conv)
    _check_fwd(y[..., keep], idx[..., keep], y_ref[..., keep], arg_ref[..., keep], pre64[..., keep, :],
               zmax[..., keep])
    assert not torch.isnan(y[..., keep]).any()
    dw, db = ops.crnn_stem_bwd(x, dy, idx, conv, POOL)
    dw_ref, db_ref = _reference_bwd(x, dy, idx)
    assert bool((dw[co] == 0).all()) and float(db[co]) == 0.0
    assert _rel(dw[keep], dw_ref[keep]) <= 1e-5 and _rel(db[keep], db_ref[keep]) <= 1e-5


@pytest.mark.gpu
def test_cuda_graph_replay_matches_eager(cuda):
    from megreader_b200 import nnops as ops
    conv = _conv(5, cuda)
    xs, dys = _inputs(6, 8, 32, 100, cuda)
    ops.crnn_stem_bwd(xs, dys, ops.crnn_stem_fwd(xs, conv, POOL, True)[1], conv, POOL)      # warm-up (scratch allocation)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y, idx = ops.crnn_stem_fwd(xs, conv, POOL, True)
        dw, db = ops.crnn_stem_bwd(xs, dys, idx, conv, POOL)
    for seed in (7, 8):
        x, dy = _inputs(seed, 8, 32, 100, cuda)
        xs.copy_(x)
        dys.copy_(dy)
        graph.replay()
        y_e, idx_e = ops.crnn_stem_fwd(x, conv, POOL, True)
        dw_e, db_e = ops.crnn_stem_bwd(x, dy, idx_e, conv, POOL)
        torch.cuda.synchronize()
        for got, want in ((y, y_e), (idx, idx_e), (dw, dw_e), (db, db_e)):
            assert torch.equal(got, want)


@pytest.mark.gpu
def test_no_grad_forward_writes_no_routing(cuda):
    from megreader_b200 import nnops as ops
    conv = _conv(9, cuda)
    x, _ = _inputs(10, 4, 32, 100, cuda)
    y, idx = ops.crnn_stem_fwd(x, conv, POOL, True)
    y0, idx0 = ops.crnn_stem_fwd(x, conv, POOL, False)
    assert idx0 is None and torch.equal(y, y0)


def _geo(**kw):
    g = dict(N=2, Cin=3, H=32, W=100, Cout=64, kh=3, kw=3, sh=1, sw=1, ph=1, pw=1, pkh=2, pkw=2, psh=2, psw=2, pph=0, ppw=0)
    g.update(kw)
    return list(g.values())


@pytest.mark.parametrize("bad", [dict(Cin=1), dict(Cin=4), dict(Cout=32), dict(kh=5, kw=5, ph=2, pw=2), dict(kw=1, pw=0),
                                 dict(sh=2), dict(ph=0, pw=0), dict(pkh=3), dict(psw=1), dict(pph=1), dict(H=1),
                                 dict(W=1)], ids=str)
def test_refused_geometry(bad):
    """Geometries the stem does not cover return MR_ERR_UNSUPPORTED before any pointer is touched (no GPU needed)."""
    L = _lib.lib()
    p = 256                                  # aligned dummy pointer: the checks come first
    assert L.mr_crnn_stem_fwd(p, p, p, *_geo(**bad), p, p, None) == _lib.MR_ERR_UNSUPPORTED
    assert L.mr_crnn_stem_bwd(p, p, p, *_geo(**bad), p, p, p, None) == _lib.MR_ERR_UNSUPPORTED


def test_bad_arguments():
    L = _lib.lib()
    p = 256
    for bad in (dict(N=-1), dict(H=0), dict(W=-2), dict(Cin=0), dict(kh=0), dict(psh=0), dict(ph=-1)):
        assert L.mr_crnn_stem_fwd(p, p, p, *_geo(**bad), p, p, None) == 4, bad        # MR_ERR_BAD_SHAPE
        assert L.mr_crnn_stem_bwd(p, p, p, *_geo(**bad), p, p, p, None) == 4, bad
    for i in range(3):                       # x, w, bias
        ptrs = [p, p, p]
        ptrs[i] = None
        assert L.mr_crnn_stem_fwd(*ptrs, *_geo(), p, p, None) == 1                    # MR_ERR_NULL_POINTER
    assert L.mr_crnn_stem_fwd(p, p, p, *_geo(), None, p, None) == 1
    for i in range(3):                       # dw, dbias, sums
        ptrs = [p, p, p]
        ptrs[i] = None
        assert L.mr_crnn_stem_bwd(p, p, p, *_geo(), *ptrs, None) == 1
    for i in range(3):                       # x, dy, idx
        ptrs = [p, p, p]
        ptrs[i] = None
        assert L.mr_crnn_stem_bwd(*ptrs, *_geo(), p, p, p, None) == 1
    assert L.mr_crnn_stem_fwd(None, None, None, *_geo(N=0), None, None, None) == 0    # empty batch: nothing to do


def _train_step(cuda, stem_on, monkeypatch, x_grad=False):
    import megreader_b200
    from megreader_b200 import crnn_engine
    from megreader_b200 import nnops as ops
    from tests.weights import crnn_batch, fill_state_dict
    megreader_b200.install_reference_api()
    import backbones
    import decoders
    bb = fill_state_dict(backbones.crnn_backbone(), "bb.").to(cuda).train()
    dec = fill_state_dict(decoders.CRNNDecoder(in_channels=512, inner_channels=256), "dec.").to(cuda).train()
    x, labels, lengths = [torch.from_numpy(a).to(cuda) for a in crnn_batch(0, 64, 256, 16, 65)]
    x.requires_grad_(x_grad)
    calls = []
    real = ops.crnn_stem_fwd
    monkeypatch.setattr(ops, "crnn_stem_fwd", (lambda *a: calls.append(1) or real(*a)) if stem_on else (lambda *a: None))
    crnn_engine.set_compute_dtype(torch.bfloat16)
    try:
        loss, _ = dec(bb(x), targets=labels, lengths=lengths, train=True)
        loss.mean().backward()
        torch.cuda.synchronize()
    finally:
        crnn_engine.set_compute_dtype(torch.float32)
        monkeypatch.setattr(ops, "crnn_stem_fwd", real)
    norms = {n: p.grad.double().norm().item() for n, p in list(bb.named_parameters()) + list(dec.named_parameters())}
    return float(loss.mean().item()), norms, len(calls), x.grad


@pytest.mark.gpu
def test_engine_step_with_and_without_stem(cuda, monkeypatch):
    loss, norms, calls, _ = _train_step(cuda, True, monkeypatch)
    loss0, norms0, _, _ = _train_step(cuda, False, monkeypatch)
    assert calls == 1
    assert abs(loss - loss0) <= 1e-3 * abs(loss0)
    for k in norms0:
        if k in ("cnn.2.0.bias", "cnn.4.0.bias", "cnn.6.0.bias"):
            continue                         # conv bias before BatchNorm: the gradient is 0 up to rounding noise
        assert abs(norms[k] - norms0[k]) <= 1e-2 * norms0[k] + 1e-6, (k, norms[k], norms0[k])


@pytest.mark.gpu
def test_engine_image_gradient_takes_unfused_branch(cuda, monkeypatch):
    _, norms, calls, xg = _train_step(cuda, True, monkeypatch, x_grad=True)
    assert calls == 0 and xg is not None and torch.isfinite(xg).all() and float(xg.abs().sum()) > 0
