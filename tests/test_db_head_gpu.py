"""GPU: the DB detector tail on csrc/db_head.cu (megreader_b200.db_head) against the float64 restatement tests/db_port.py, the
reference's framework composition, and tests/golden/seg_detector_ref.npz."""
import numpy as np
import pytest
import torch

from tests import db_port
from tests.db_data import db_batch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


@pytest.fixture(autouse=True)
def _no_tf32():
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def _db():
    from megreader_b200 import db_head
    return db_head


def _decoders():
    import megreader_b200.refapi.decoders as decoders      # by package path: `decoders` may be the reference's in this process
    return decoders


def _close(got, ref, rtol, what=""):
    got, ref = got.detach().double(), ref.detach().double()
    err = float((got - ref).abs().max())
    scale = float(ref.abs().max())
    assert err <= rtol * max(scale, 1e-30), "%s: max err %.3e vs max |ref| %.3e" % (what, err, scale)


# ------------------------------------------------------------------------------------------------------------- 1. step
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("adaptive", [True, False])
def test_step_function(dtype, adaptive):
    g = torch.Generator(device=DEV).manual_seed(1)
    zb = (3 * torch.randn(2, 1, 33, 47, device=DEV, generator=g)).to(dtype).requires_grad_(True)
    zt = (torch.randn(2, 1, 33, 47, device=DEV, generator=g)).to(dtype).requires_grad_(True) if adaptive else None
    out = _db().step_function(zb, zt, 50.0)
    gs = [torch.randn(2, 1, 33, 47, device=DEV, generator=g) for _ in range(3)]
    zb64 = zb.detach().double().requires_grad_(True)
    zt64 = zt.detach().double().requires_grad_(True) if adaptive else None
    ref = db_port.step(zb64, zt64, 50.0)
    n = 3 if adaptive else 1
    for i in range(n):
        assert out[i].dtype == torch.float32
        # the step function multiplies the fp32 rounding of binary - thresh (2^-24 each) by up to k / 4
        _close(out[i].detach(), ref[i], 1e-6 if i < 2 else 2 * 2 ** -24 * 50.0 / 4 + 1e-6, "map %d" % i)
    sum((o * gg).sum() for o, gg in zip(out[:n], gs)).backward()
    sum((o * gg.double()).sum() for o, gg in zip(ref[:n], gs)).backward()
    assert zb.grad.dtype == dtype
    tol = 1e-5 if dtype == torch.float32 else 8e-3        # bf16: the gradient is rounded once to bf16
    _close(zb.grad, zb64.grad, tol, "d zb")
    if adaptive:
        _close(zt.grad, zt64.grad, tol, "d zt")
    else:
        assert out[1] is None and out[2] is None


# ------------------------------------------------------------------------------------------------------------- 2. loss
def _case(N, H, W, seed, quantise=False, soft=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    b = {k: torch.from_numpy(v).to(DEV) for k, v in db_batch(seed, N, H, W).items()}
    z = [3 * torch.randn(N, 1, H, W, device=DEV, generator=g) for _ in range(3)]
    if quantise:                                     # bf16 logits: binary takes few distinct values, many ties at tau
        z = [t.bfloat16().float() for t in z]
    maps = [torch.sigmoid(t) for t in z]
    maps[1] = maps[1] * 0.8 + 0.1
    if soft:
        b["gt"] = torch.where(torch.rand(b["gt"].shape, device=DEV, generator=g) < 0.2,
                              torch.rand(b["gt"].shape, device=DEV, generator=g), b["gt"])
    return maps, b


def _run_fused(maps, b, **kw):
    x = [m.clone().requires_grad_(True) for m in maps]
    out = _db().l1_balance_ce_loss(*x, b["gt"], b["mask"], b["thresh_map"], b["thresh_mask"], **kw)
    out[0].backward()
    return [o.detach() for o in out], [t.grad for t in x]


def _run_port(maps, b, **kw):
    x = [m.double().requires_grad_(True) for m in maps]
    pred = dict(binary=x[0], thresh=x[1], thresh_binary=x[2])
    loss, m = db_port.l1_balance_ce(pred, b, **kw)
    loss.backward()
    return [loss.detach(), m["bce_loss"].detach(), m["thresh_loss"].detach(), m["l1_loss"].detach()], [t.grad for t in x]


def _scalar_close(a, b, rtol=1e-5, what=""):
    a, b = float(a), float(b)
    assert abs(a - b) <= rtol * abs(b) + 1e-12, "%s: %r vs %r" % (what, a, b)


def _check_loss(maps, b, tie_free=True, **kw):
    got, g = _run_fused(maps, b, **kw)
    ref, gr = _run_port(maps, b, **kw)
    for i, name in enumerate(("loss", "bce", "dice", "l1")):
        if np.isnan(float(ref[i])):
            assert np.isnan(float(got[i])), name
        else:
            _scalar_close(got[i], ref[i], 1e-5, name)
    if not np.isnan(float(ref[3])):
        _close(g[1], gr[1], 1e-5, "d thresh")
    _close(g[2], gr[2], 1e-5, "d thresh_binary")
    if tie_free:
        _close(g[0], gr[0], 1e-5, "d binary")
    else:
        # per tie class: pixels with the same binary value and the same weights share one gradient sum
        p = maps[0].reshape(-1)
        key = torch.stack([p.double(), b["gt"].reshape(-1).double(), b["mask"].reshape(-1).double()], 1)
        _, inv = torch.unique(key, dim=0, return_inverse=True)
        sg = torch.zeros(int(inv.max()) + 1, dtype=torch.float64, device=DEV).index_add_(0, inv, g[0].reshape(-1).double())
        sr = torch.zeros_like(sg).index_add_(0, inv, gr[0].reshape(-1).double())
        _close(sg, sr, 1e-5, "d binary per tie class")
    return got


@pytest.mark.parametrize("N,H,W", [(2, 40, 40), (4, 640, 640)])
def test_loss_vs_port(N, H, W):
    maps, b = _case(N, H, W, 3)
    _check_loss(maps, b)


@pytest.mark.parametrize("N,H,W", [(2, 40, 40), (4, 640, 640)])
def test_loss_vs_port_bf16_ties(N, H, W):
    maps, b = _case(N, H, W, 4, quantise=True)
    _check_loss(maps, b, tie_free=False)


def test_loss_edge_cases():
    maps, b = _case(2, 40, 40, 5)
    nb = dict(b, gt=torch.zeros_like(b["gt"]))                                   # no positives: k = 0, bce = 0
    got = _check_loss(maps, nb)
    assert float(got[1]) == 0.0
    _check_loss(maps, dict(b, gt=torch.ones_like(b["gt"])))                      # no negatives
    few = torch.zeros_like(b["gt"])
    few[:, :, 5:30, 5:30] = 1                                                    # 39 % positive: k clamped by #neg
    _check_loss(maps, dict(b, gt=few))
    got = _check_loss(maps, dict(b, mask=torch.zeros_like(b["mask"])))           # everything masked out
    assert float(got[1]) == 0.0
    maps_s, b_s = _case(2, 40, 40, 6, soft=True)                                 # soft (non-binary) gt
    _check_loss(maps_s, b_s)
    got = _check_loss(maps, dict(b, thresh_mask=torch.zeros_like(b["thresh_mask"])))   # empty thresh_mask -> NaN
    assert np.isnan(float(got[0])) and np.isnan(float(got[3]))


# ----------------------------------------------------------------------------------------------------- 3. the select
def _bce_vs_topk(p, gt, mask, ratio):
    """bce metric of the fused loss vs the framework composition (torch.topk over the broadcast values)."""
    z = torch.full_like(p, 0.5)
    m = torch.ones_like(mask)
    got = _db().l1_balance_ce_loss(p, z, z, gt, mask, mask, m, negative_ratio=ratio)[1]
    ref = _decoders().BalanceCrossEntropyLoss(negative_ratio=ratio)(p, gt, mask)
    _scalar_close(got, ref, 2e-6, "bce")


def test_select_vs_topk():
    g = torch.Generator(device=DEV).manual_seed(8)
    H, W = 64, 96
    p = torch.rand(1, 1, H, W, device=DEV, generator=g).clamp(1e-6, 1 - 1e-6)
    mask = torch.ones(1, H, W, device=DEV)
    gt = torch.zeros(1, 1, H, W, device=DEV)
    _bce_vs_topk(p, gt, mask, 3.0)                                               # k = 0
    one = gt.clone(); one[0, 0, 3, 4] = 1
    _bce_vs_topk(p, one, mask, 1.0)                                              # k = 1
    _bce_vs_topk(p, one, mask, 1e9)                                              # k = #neg = all but one value
    many = (torch.rand(1, 1, H, W, device=DEV, generator=g) < 0.4).float()
    _bce_vs_topk(p, many, mask, 3.0)                                             # k clamped to #neg
    tied = torch.tensor([0.1, 0.3, 0.5, 0.7], device=DEV)[torch.randint(0, 4, (1, 1, H, W), device=DEV, generator=g)]
    sparse = (torch.rand(1, 1, H, W, device=DEV, generator=g) < 0.1).float()
    _bce_vs_topk(tied, sparse, mask, 3.0)                                        # heavily tied
    binades = 10 ** (-30 * torch.rand(1, 1, H, W, device=DEV, generator=g))     # 1e-30 .. 1
    _bce_vs_topk(binades.clamp(max=1 - 1e-7), sparse, mask, 3.0)                 # values spanning many binades
    N = 3                                                                        # the N x N broadcast
    p3 = torch.rand(N, 1, H, W, device=DEV, generator=g).clamp(1e-6, 1 - 1e-6)
    gt3 = (torch.rand(N, 1, H, W, device=DEV, generator=g) < 0.1).float()
    m3 = (torch.rand(N, H, W, device=DEV, generator=g) < 0.9).float()
    _bce_vs_topk(p3, gt3, m3, 3.0)


# ----------------------------------------------------------------------------------------- 4. graphs and determinism
def test_graph_capture_and_determinism():
    maps, b = _case(2, 96, 128, 9)
    maps2, b2 = _case(2, 96, 128, 10)
    b2["gt"][:, :, :20] = 1                                                      # a different positive count
    assert int(b2["gt"].sum()) != int(b["gt"].sum())
    e1, g1 = _run_fused(maps, b)
    e1b, g1b = _run_fused(maps, b)
    for x, y in zip(e1 + g1, e1b + g1b):
        assert torch.equal(x, y)
    e2, g2 = _run_fused(maps2, b2)
    x = [m.clone().requires_grad_(True) for m in maps]
    sb = {k: v.clone() for k, v in b.items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for t in x:
                t.grad = None
            out = _db().l1_balance_ce_loss(*x, sb["gt"], sb["mask"], sb["thresh_map"], sb["thresh_mask"])
            out[0].backward()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    for t in x:
        t.grad = None
    with torch.cuda.graph(graph):
        out = _db().l1_balance_ce_loss(*x, sb["gt"], sb["mask"], sb["thresh_map"], sb["thresh_mask"])
        out[0].backward()
    for src, tgt in ((maps2, b2), (maps, b)):
        with torch.no_grad():
            for t, m in zip(x, src):
                t.copy_(m)
            for k in sb:
                sb[k].copy_(tgt[k])
        graph.replay()
        torch.cuda.synchronize()
        want_o, want_g = (e2, g2) if src is maps2 else (e1, g1)
        for o, w in zip(out, want_o):
            assert torch.equal(o.detach(), w)
        for t, w in zip(x, want_g):
            assert torch.equal(t.grad, w)


# ------------------------------------------------------------------------------------------- 5. SegDetector on golden
def _golden_run(engine):
    from tests.make_db_golden import GOLD, SALT, batch, features
    from tests.weights import fill_state_dict
    gold = dict(np.load(GOLD))
    d = _decoders()
    from megreader_b200.refapi.decoders.seg_detector_loss import L1BalanceCELoss
    head = fill_state_dict(d.SegDetector(adaptive=True, k=50, in_channels=[64, 128, 256, 512]), SALT).to(DEV).train()
    if engine:
        from megreader_b200 import conv_engine
        assert conv_engine.use_engine_convs(head) > 0
    feats = [torch.from_numpy(f).float().to(DEV).requires_grad_(True) for f in features()]
    b = {k: torch.from_numpy(v).float().to(DEV) for k, v in batch().items()}
    pred = head(feats, training=True)
    loss, metrics = L1BalanceCELoss()(pred, b)
    loss.backward()
    torch.cuda.synchronize()
    return gold, pred, loss, metrics, feats


def test_seg_detector_golden_library_fp32():
    gold, pred, loss, metrics, feats = _golden_run(False)
    _scalar_close(loss, gold["loss"], 1e-4, "loss")
    for k, v in metrics.items():
        _scalar_close(v, gold["m_" + k], 1e-4, k)
    for k, v in pred.items():
        _close(v.detach(), torch.from_numpy(gold["train_" + k]).to(DEV), 1e-4, k)
    for i, f in enumerate(feats):
        _close(f.grad, torch.from_numpy(gold["gf%d" % i]).to(DEV), 1e-4, "grad c%d" % (i + 2))


def _cos(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a @ b) / (a.norm() * b.norm()))


def test_seg_detector_golden_engine_bf16():
    gold, pred, loss, metrics, feats = _golden_run(True)
    assert pred["binary"].dtype == torch.float32
    assert abs(float(loss) - float(gold["loss"])) <= 5e-2 * abs(float(gold["loss"]))
    for i, f in enumerate(feats):
        assert _cos(f.grad, torch.from_numpy(gold["gf%d" % i]).to(DEV)) > 0.9, i


# ----------------------------------------------------------------------------------------- 6. the seg_detector_db step
def test_seg_detector_db_step_engine_vs_library():
    """As tests/test_trunks_engine_gpu.py: one model, library fp32 convolutions first, then every eligible convolution on the
    engine (bf16).  BatchNorm on running statistics: at N = 2 the batch statistics of the 8 x 8 stage-5 maps turn bf16 rounding
    into O(1) changes of the normalised activations, a property of the model at this batch size, not of the kernels."""
    import bench_trunks
    from megreader_b200 import conv_engine
    torch.manual_seed(0)
    net, n = bench_trunks.build(6, DEV, engine=False)
    assert n == 0
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eval()
    x, lab = bench_trunks.synth_db(3, 2, (256, 256))
    x, lab = x.to(DEV), {k: v.to(DEV) for k, v in lab.items()}
    state = {k: v.clone() for k, v in net.state_dict().items()}

    def run():
        for p in net.parameters():
            p.grad = None
        loss, pred = net(x, lab, None)
        loss.backward()
        torch.cuda.synchronize()
        g = {k: p.grad.detach().float().clone() for k, p in net.named_parameters() if p.grad is not None}
        net.load_state_dict(state)
        return float(loss), g
    l_lib, g_lib = run()
    assert conv_engine.use_engine_convs(net, wgrad_side_stream=False) > 60
    try:
        l_eng, g_eng = run()
    finally:
        conv_engine.restore_library_convs(net)
    assert np.isfinite(l_lib) and abs(l_eng - l_lib) <= 5e-2 * abs(l_lib), (l_eng, l_lib)
    assert set(g_eng) == set(g_lib) and all(bool(torch.isfinite(v).all()) for v in g_eng.values())
    checked = 0
    for k, r in g_lib.items():
        if r.numel() >= 64 * 64 and float(r.norm()) > 1e-6:
            assert _cos(g_eng[k], r) > 0.9, (k, _cos(g_eng[k], r))
            checked += 1
    assert checked > 20
