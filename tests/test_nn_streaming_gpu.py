"""GPU: the streaming kernels of the CRNN step (csrc/nn_kernels.cu) against float64 computations of the same operation on
the same (already rounded) inputs, at the CRNN layer shapes and at every host dispatch variant that tests/nn_variants.py
restates: training BatchNorm forward / backward (statistics, running buffers, the fused bias gradient), bias + ReLU +
max-pool forward / backward, column sums, bias + activation, casts, im2col / col2im, layout conversion and the LSTM
cell.  Where a case names its kernels, torch.profiler checks them once per kernel.

KERNELS (every kernel some case below expects) is read by tests/test_kernel_inventory.py without a GPU."""
import copy
import warnings

import pytest
import torch
import torch.nn.functional as F

from tests import nn_variants as nv
from tests.wgmma_variants import launched_kernels

F32, BF16 = torch.float32, torch.bfloat16
NAME = {F32: "float", BF16: "bf16"}
U = 2.0 ** -24                                       # fp32 unit roundoff
EPS = 1e-5
MOMENTUM = float(torch.tensor(0.1, dtype=torch.float32))   # the fp32 momentum the kernel receives

# ---------------------------------------------------------------- cases (module level: the inventory reads them)
BN_SHAPES = {"L2": (512, 256), "L4": (260, 512), "L6": (65, 512)}     # (pixels per image, C) of the BatchNorm layers
BN_CASES = [(layer, n, dt, ratio) for layer in BN_SHAPES for n in (512, 1) for dt in (F32, BF16)
            for ratio in (0, 1, 10, 100, 1000)]
# (dtype, rows, C, want_dbias): bn_apply_kernel / bn_bwd_apply_kernel (channel-vector count does not divide 256; fp32
# C = 24 shares the channel vector across the two in-flight vectors, bf16 C = 40 does not), the fp64-atomic statistics
# (2C > 4096), no bias gradient
BN_EDGE = [(F32, 262144, 24, True), (BF16, 262144, 40, True), (BF16, 4096, 2056, True), (F32, 3000, 64, False),
           (BF16, 3000, 40, False)]

CRNN_POOLS = {"L1": (16, 128, 128, (2, 2), (2, 2), (0, 0)), "L3": (8, 64, 256, (2, 2), (2, 1), (0, 1)),
              "L5": (4, 65, 512, (2, 2), (2, 1), (0, 1))}             # (H, W, C, window, stride, padding) of the pool input
# (id, dtype, N, H, W, C, k, s, p, want_dbias, special)
POOL_CASES = [("crnn-%s" % name, BF16, 512) + g + (True, None) for name, g in CRNN_POOLS.items()]
POOL_CASES += [("crnn-%s" % name, F32, 8) + g + (True, None) for name, g in CRNN_POOLS.items()]
for _dt in (F32, BF16):
    POOL_CASES += [
        ("2x2-stride1", _dt, 3, 9, 11, 64, (2, 2), (1, 1), (0, 0), True, None),        # pool_bwd_rows_kernel
        ("2x2-vpad", _dt, 3, 10, 12, 32, (2, 2), (2, 2), (1, 0), True, None),          # pool_bwd_rows_kernel
        ("3x3-tiled", _dt, 4, 12, 15, 64, (3, 3), (3, 3), (0, 0), True, None),         # generic tiled, partials
        ("3x3-tiled-nodbias", _dt, 4, 12, 15, 64, (3, 3), (3, 3), (0, 0), False, None),
        ("3x3-overlap", _dt, 4, 11, 13, 64, (3, 3), (2, 2), (1, 1), True, None),       # generic gather, partials
        ("3x3-overlap-c24", _dt, 4, 11, 13, 24 if _dt == F32 else 48, (3, 3), (2, 2), (1, 1), True, None),  # colsum
        ("2x2-c24", _dt, 5, 8, 10, 24 if _dt == F32 else 40, (2, 2), (2, 2), (0, 0), True, None),
        ("ties-inf", _dt, 6, 8, 10, 64, (2, 2), (2, 2), (0, 0), True, "ties_inf"),
        ("ties-inf-3x3", _dt, 6, 9, 12, 64, (3, 3), (2, 2), (1, 1), True, "ties_inf"),
        ("nan", _dt, 6, 8, 10, 64, (2, 2), (2, 2), (0, 0), True, "nan"),
        ("nan-3x3", _dt, 6, 9, 12, 64, (3, 3), (2, 2), (1, 1), True, "nan"),
        ("nan-crnn-L3", _dt, 4, 8, 64, 256, (2, 2), (2, 1), (0, 1), True, "nan"),
    ]
COLSUM_CASES = [(F32, 20000, 256), (BF16, 20000, 256), (F32, 500, 38), (BF16, 500, 38), (BF16, 4096, 2056)]
BIAS_ACT_CASES = [(dt, C, relu) for dt in (F32, BF16) for C in (64, 38) for relu in (False, True)]
CAST_PAIRS = [(a, b) for a in (F32, BF16) for b in (F32, BF16)]
IM2COL_CASES = [(F32, 2, 6, 9, 3, 3, 3, 1, 1, 27), (BF16, 2, 6, 9, 3, 3, 3, 1, 1, 32), (F32, 2, 6, 9, 8, 3, 3, 1, 1, 76),
                (BF16, 3, 5, 7, 16, 3, 3, 1, 1, 152), (F32, 2, 4, 65, 512, 2, 2, 0, 0, 2048)]
LSTM_CASES = [(dt, ndir, prev, H, B) for dt in (F32, BF16) for ndir in (1, 2) for prev in (False, True)
              for H in (64, 256) for B in (1, 500)]


def _collect():
    ks = set()
    for layer, n, dt, _ in BN_CASES:
        hw, C = BN_SHAPES[layer]
        ks |= nv.plan("mr_bn_train_fwd", NAME[dt], n * hw, C) | nv.plan("mr_bn_train_bwd", NAME[dt], n * hw, C)
        ks |= nv.plan("mr_bn_apply", NAME[dt], n * hw, C)
    for dt, rows, C, want in BN_EDGE:
        ks |= nv.plan("mr_bn_train_fwd", NAME[dt], rows, C) | nv.plan("mr_bn_apply", NAME[dt], rows, C)
        ks |= nv.plan("mr_bn_train_bwd", NAME[dt], rows, C, want_dbias=want)
    for _, dt, N, H, W, C, k, s, p, want, _ in POOL_CASES:
        ks |= nv.plan("mr_bias_relu_pool_fwd", NAME[dt], N, H, W, C, k, s, p)
        ks |= nv.plan("mr_bias_relu_pool_bwd", NAME[dt], N, H, W, C, k, s, p, want_dbias=want)
    for dt, rows, C in COLSUM_CASES:
        ks |= nv.plan("mr_colsum", NAME[dt], rows, C)
    for dt, C, _ in BIAS_ACT_CASES:
        ks |= nv.plan("mr_bias_act", NAME[dt], 300, C)
    for a, b in CAST_PAIRS:
        ks |= nv.plan("mr_cast", NAME[a], NAME[b])
    for dt, N, H, W, C, kh, kw, ph, pw, Kp in IM2COL_CASES:
        ks |= nv.plan("mr_im2col_nhwc", NAME[dt], C, Kp)
        if C % nv.VN[NAME[dt]] == 0 and Kp % nv.VN[NAME[dt]] == 0:
            ks |= nv.plan("mr_col2im_nhwc", NAME[dt], C, Kp)
    for dt in (F32, BF16):
        ks |= nv.plan("mr_nchw_to_nhwc", NAME[dt]) | nv.plan("mr_nhwc_to_nchw", NAME[dt])
        ks |= nv.plan("mr_lstm_cell_fwd", NAME[dt]) | nv.plan("mr_lstm_cell_bwd", NAME[dt])
    return frozenset(ks)


KERNELS = _collect()


# ---------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def ops(cuda):
    from megreader_b200 import nnops
    return nnops


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


_CHECKED = set()
_NN = nv.REACHABLE | frozenset(nv.COVERED_ELSEWHERE)


def run(expected, fn):
    """fn() must launch exactly the nn_kernels.cu kernels in `expected`; checked under torch.profiler only while some of
    them have not been seen yet.  As in wgmma_variants.run_variant, a trace without the expected records only warns: long
    profiler sessions were seen to lose the library's kernel records.  -> fn's result."""
    expected = frozenset(expected)
    if expected <= _CHECKED:
        return fn()
    result, names = launched_kernels(fn)
    seen = {nv.nn_normalise(n) for n in names} & _NN
    assert seen <= expected, "expected %s to run, the profiler saw %s" % (sorted(expected), sorted(seen))
    if seen != expected:
        warnings.warn("torch.profiler recorded no record for %s: not checked" % sorted(expected - seen))
    _CHECKED.update(seen)
    return result


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ulp(v, dtype):
    """one ulp of dtype at |v| (0 has none: an exact zero must stay zero)"""
    bits = 23 if dtype == F32 else 7
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -126)))
    return torch.where(v == 0, torch.zeros_like(v), torch.exp2(e - bits))


def _within(got, want, bound, what):
    got, want = got.double(), want.double()
    bad = ~((got - want).abs() <= bound)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError("%s: %d of %d outside the bound; first at flat %d: got %r, want %r, bound %.3g"
                             % (what, int(bad.sum()), bad.numel(), i, float(got.reshape(-1)[i]),
                                float(want.reshape(-1)[i]), float(bound.reshape(-1)[i])))


def _same_bits_or_both_nan(got, want, what):
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), "%s: NaN at %d positions, want %d" % (what, int(gn.sum()), int(wn.sum()))
    assert torch.equal(got[~gn], want[~wn]), what


# ---------------------------------------------------------------- BatchNorm
def _bn_inputs(rows, C, ratio, dtype, seed):
    g = _gen(seed)
    std = torch.rand(C, generator=g, device="cuda") * 1.5 + 0.5
    z = (torch.randn(rows, C, generator=g, device="cuda") * std + ratio * std).to(dtype)
    bias = torch.randn(C, generator=g, device="cuda") * 0.1
    gamma = torch.rand(C, generator=g, device="cuda") + 0.5
    beta = torch.randn(C, generator=g, device="cuda")
    rm = torch.randn(C, generator=g, device="cuda")
    rv = torch.rand(C, generator=g, device="cuda") + 0.5
    dy = torch.randn(rows, C, generator=g, device="cuda").to(dtype)
    return z, bias, gamma, beta, rm, rv, dy


def _bn_check(ops, dtype, rows, C, ratio, seed, want_dbias=True):
    T, sms = NAME[dtype], _sms()
    z, bias, gamma, beta, rm, rv, dy = _bn_inputs(rows, C, ratio, dtype, seed)
    rm0, rv0 = rm.double(), rv.double()
    y, mean, invstd = run(nv.plan("mr_bn_train_fwd", T, rows, C, sms=sms),
                          lambda: ops.bn_train_fwd(z, bias, gamma, beta, rm, rv, MOMENTUM, EPS))
    # float64 reference on the values the kernels read: the fp32 sum z + b (what an unfused conv bias would store)
    x = (z.float() + bias).double()
    m64 = x.mean(0)
    var64 = x.var(0, unbiased=False)
    inv64 = (var64 + EPS).rsqrt()
    xhat = (x - m64) * inv64
    g64, b64 = gamma.double(), beta.double()
    y64 = xhat * g64 + b64
    unb = var64 * rows / (rows - 1) if rows > 1 else var64
    rm64 = (1 - MOMENTUM) * rm0 + MOMENTUM * m64
    rv64 = (1 - MOMENTUM) * rv0 + MOMENTUM * unb
    sd = var64.sqrt()
    # statistics: fp32 rounding of the stored values, plus a 1e-6 relative summation allowance; the fp32 sums of x and
    # x^2 (without a shift) lose ~1e-4 relative variance at mean/std = 100 and everything at 1000
    _within(mean, m64, 2 * U * m64.abs() + 1e-6 * sd, "mean")
    _within(invstd, inv64, 2e-6 * inv64, "invstd")
    _within(rm, rm64, 4 * U * (rm64.abs() + rm0.abs()) + 1e-6 * MOMENTUM * sd, "running_mean")
    _within(rv, rv64, 2e-6 * rv64.abs() + 4 * U * rv0.abs(), "running_var")
    # y = z * sc + sh with sc = invstd * gamma, sh = (b - mean) * sc + beta: a few fp32 roundings of the terms it adds,
    # and the statistics' own allowances (invstd relative, mean 1e-6 sd)
    cond = (z.double().abs() + (bias.double() - m64).abs()) * inv64 * g64.abs() + b64.abs()
    yb = 16 * U * (cond + y64.abs()) + 4e-6 * (xhat * g64).abs() + 1e-6 * g64.abs() * inv64 * sd
    if dtype == BF16:
        yb = yb + 2.0 ** -8 * y64.abs()
    _within(y, y64, yb, "y")

    dx, dgamma, dbeta, dbias = run(nv.plan("mr_bn_train_bwd", T, rows, C, want_dbias=want_dbias, sms=sms),
                                   lambda: ops.bn_train_bwd(dy, z, bias, mean, invstd, gamma, want_dbias=want_dbias))
    d = dy.double()
    k1, k2 = d.mean(0), (d * xhat).mean(0)
    A = g64 * inv64
    dx64 = A * (d - k1 - xhat * k2)
    m_abs = d.abs().mean(0)
    ratio_c = m64.abs() / sd
    dxb = A.abs() * (16 * U * d.abs() + 2.0 ** -18 * m_abs * (1 + xhat.abs()) * (1 + ratio_c)) + \
        4e-6 * A.abs() * (d.abs() + xhat.abs() * k2.abs())
    if dtype == BF16:
        dxb = dxb + 2.0 ** -8 * dx64.abs()
    _within(dx, dx64, dxb, "dx")
    _within(dbeta, d.sum(0), 1e-6 * d.abs().sum(0), "dbeta")
    _within(dgamma, (d * xhat).sum(0), (1e-6 + 2.0 ** -18 * ratio_c) * (d.abs() * (1 + xhat.abs())).sum(0) +
            4e-6 * (d * xhat).sum(0).abs(), "dgamma")
    if want_dbias:
        dxs = dx.double()
        _within(dbias, dxs.sum(0), 1e-6 * dxs.abs().sum(0), "dbias (sum of the stored dx)")
    else:
        assert dbias is None

    # eval-mode apply with the batch statistics: the same map y = z * sc + sh
    ye = run(nv.plan("mr_bn_apply", T, rows, C), lambda: ops.bn_apply(z, bias, mean, invstd, gamma, beta))
    assert torch.equal(ye, y), "bn_apply differs from the training forward's apply with the same statistics"


@pytest.mark.gpu
@pytest.mark.parametrize("layer,n,dtype,ratio", BN_CASES, ids=lambda v: str(v).replace("torch.", ""))
def test_batchnorm_crnn_shapes(cuda, ops, layer, n, dtype, ratio):
    hw, C = BN_SHAPES[layer]
    _bn_check(ops, dtype, n * hw, C, ratio, seed=1000 * list(BN_SHAPES).index(layer) + 10 * n + ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,rows,C,want_dbias", BN_EDGE, ids=lambda v: str(v).replace("torch.", ""))
@pytest.mark.parametrize("ratio", [0, 1000])
def test_batchnorm_dispatch_edges(cuda, ops, dtype, rows, C, want_dbias, ratio):
    T = NAME[dtype]
    cv = C // nv.VN[T]
    if 256 % cv:
        assert "bn_bwd_apply_kernel<%s>" % T in nv.plan("mr_bn_train_bwd", T, rows, C)
        if rows >= 100000:
            br = nv.bn_bwd_apply_branches(T, rows, C, sms=_sms())
            assert br >= ({"two"} if C == 24 else {"differs"}), br
    _bn_check(ops, dtype, rows, C, ratio, seed=rows + C, want_dbias=want_dbias)


# ---------------------------------------------------------------- bias + ReLU + max-pool
def _pool_check(ops, dtype, N, H, W, C, k, s, p, want_dbias, special, seed):
    from megreader_b200.nnops import pool_out
    T, sms = NAME[dtype], _sms()
    Ho, Wo = pool_out(H, W, k, s, p)
    g = _gen(seed)
    z = torch.randn(N, H, W, C, generator=g, device="cuda")
    bias = torch.randn(C, generator=g, device="cuda") * 0.5
    if special == "ties_inf":
        bias = torch.round(bias * 4) / 4
        z[0] = -z[0].abs() - 1 - bias.clamp_min(0)                # every window of image 0 is negative: the zeros tie
        z[1:] = torch.round(z[1:] * 2) / 2                        # z + b on a 1/4 grid: equal values inside windows
        flat = z.view(-1)
        pick = torch.randint(0, flat.numel(), (flat.numel() // 97,), generator=g, device="cuda")
        flat[pick[0::2]] = float("inf")
        flat[pick[1::2]] = float("-inf")
    elif special == "nan":
        flat = z.view(-1)
        pick = torch.randint(0, flat.numel(), (flat.numel() // 61,), generator=g, device="cuda")
        flat[pick] = float("nan")
    z = z.to(dtype).view(N * H * W, C)
    dy = torch.randn(N, Ho, Wo, C, generator=g, device="cuda").to(dtype)

    y, idx = run(nv.plan("mr_bias_relu_pool_fwd", T, N, H, W, C, k, s, p),
                 lambda: ops.bias_relu_pool_fwd(z, bias, N, H, W, C, k, s, p))
    # reference: the unfused bias + ReLU stored in T, then ATen's max-pool (which keeps NaN) in float64
    act = F.relu(z.float() + bias).to(dtype).double().view(N, H, W, C).permute(0, 3, 1, 2).requires_grad_(True)
    y64, ind = F.max_pool2d(act, k, s, p, return_indices=True)
    _same_bits_or_both_nan(y.double(), y64.detach().permute(0, 2, 3, 1), "pooled y")
    # the routing byte = (i, j) of ATen's arg-max inside the window (first maximum); a NaN window's byte routes nothing
    ho = torch.arange(Ho, device="cuda").view(1, 1, Ho, 1)
    wo = torch.arange(Wo, device="cuda").view(1, 1, 1, Wo)
    i = ind // W - (ho * s[0] - p[0])
    j = ind % W - (wo * s[1] - p[1])
    num = ~torch.isnan(y)
    assert torch.equal(idx.long()[num], (i * k[1] + j).permute(0, 2, 3, 1)[num]), "arg-max bytes differ from ATen's"

    dz, dbias = run(nv.plan("mr_bias_relu_pool_bwd", T, N, H, W, C, k, s, p, want_dbias=want_dbias, sms=sms),
                    lambda: ops.bias_relu_pool_bwd(dy, y, idx, N, H, W, C, k, s, p, want_dbias=want_dbias))
    # float64 gradient routed by ATen's max-pool backward; ReLU' through the pooled value (a NaN passes nothing)
    gy = dy.double().permute(0, 3, 1, 2) * (y64.detach() > 0)
    (dz64,) = torch.autograd.grad(y64, act, gy, retain_graph=True)
    (mag,) = torch.autograd.grad(y64, act, gy.abs())
    dz64 = dz64.permute(0, 2, 3, 1).reshape(N * H * W, C)
    mag = mag.permute(0, 2, 3, 1).reshape(N * H * W, C)
    # one T ulp of the sum, plus the fp32 accumulation of up to kh*kw overlapping windows
    _within(dz, dz64, _ulp(dz64, dtype) + k[0] * k[1] * U * mag, "dz (one %s ulp)" % T)
    if want_dbias:
        dzs = dz.double()
        _within(dbias, dzs.sum(0), 1e-6 * dzs.abs().sum(0), "dbias (sum of the stored dz)")
    else:
        assert dbias is None


@pytest.mark.gpu
@pytest.mark.parametrize("case", POOL_CASES, ids=lambda c: "%s-%s" % (c[0], NAME[c[1]]))
def test_bias_relu_pool(cuda, ops, case):
    name, dtype, N, H, W, C, k, s, p, want_dbias, special = case
    _pool_check(ops, dtype, N, H, W, C, k, s, p, want_dbias, special, seed=len(name) * 131 + C + N)


# ---------------------------------------------------------------- colsum, bias_act, cast, im2col / col2im, layout
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,rows,C", COLSUM_CASES, ids=str)
def test_colsum(cuda, ops, dtype, rows, C):
    a = torch.randn(rows, C, generator=_gen(rows + C), device="cuda").to(dtype)
    out = run(nv.plan("mr_colsum", NAME[dtype], rows, C, sms=_sms()), lambda: ops.colsum(a))
    a64 = a.double()
    _within(out, a64.sum(0), 1e-6 * a64.abs().sum(0), "colsum")
    acc = torch.ones(C, device="cuda")
    ops.colsum(a, out=acc, accumulate=True)
    _within(acc, a64.sum(0) + 1, 1e-6 * (a64.abs().sum(0) + 1), "colsum accumulate")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,C,relu", BIAS_ACT_CASES, ids=str)
def test_bias_act(cuda, ops, dtype, C, relu):
    g = _gen(C)
    x = torch.randn(300, C, generator=g, device="cuda").to(dtype)
    b = torch.randn(C, generator=g, device="cuda")
    y = run(nv.plan("mr_bias_act", NAME[dtype], 300, C), lambda: ops.bias_act(x, b, relu=relu))
    ref = x.float() + b                                          # one fp32 rounding of the sum, then one to T
    ref = (ref.relu() if relu else ref).to(dtype)
    assert torch.equal(y, ref)
    r64 = x.double() + b.double()
    r64 = r64.clamp_min(0) if relu else r64
    _within(y, r64, _ulp(r64, dtype) + _ulp(r64, F32), "bias_act vs float64")


def _cast_inputs(src):
    g = _gen(7)
    v = [torch.randn(4096, generator=g, device="cuda") * 3]
    if src == F32:
        base = torch.randn(512, generator=g, device="cuda").to(BF16).float()
        half = torch.exp2(torch.floor(torch.log2(base.abs().clamp_min(2.0 ** -120))) - 8) * base.sign()
        v += [base + half, base - half,                                      # exact bf16 ties: round half to even
              torch.tensor([3.4e38, -3.4e38, 3.3961e38, float("inf"), float("-inf"), float("nan"), 0.0, -0.0,
                            1e-40, -1e-40, 1.5e-45, 2.0 ** -133, 1.1754942e-38, 2.0 ** -126], device="cuda")]
    else:
        v += [torch.tensor([float("inf"), float("-inf"), float("nan"), 0.0, -0.0, 2.0 ** -133, -(2.0 ** -127),
                            3.3895e38], device="cuda")]
    return torch.cat(v).to(src)


@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", CAST_PAIRS, ids=str)
def test_cast(cuda, ops, src, dst):
    """bit-equal to Tensor.to (NaN compared as NaN: the device conversion writes its canonical NaN)"""
    from megreader_b200 import _lib
    x = _cast_inputs(src)
    y = torch.empty(x.shape, dtype=dst, device="cuda")
    run(nv.plan("mr_cast", NAME[src], NAME[dst]),
        lambda: _lib.check(_lib.lib().mr_cast(x.data_ptr(), ops.code(src), x.numel(), ops.code(dst), y.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream), "cast"))
    want = x.to(dst)
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(y), nan)
    ib = torch.int32 if dst == F32 else torch.int16
    assert torch.equal(y[~nan].view(ib), want[~nan].view(ib)), "cast bits differ from Tensor.to"


@pytest.mark.gpu
@pytest.mark.parametrize("case", IM2COL_CASES, ids=lambda c: "x".join(map(str, c[1:])) + "-" + NAME[c[0]])
def test_im2col_col2im(cuda, ops, case):
    from megreader_b200 import _lib
    dtype, N, H, W, C, kh, kw, ph, pw, Kp = case
    T = NAME[dtype]
    g = _gen(C + Kp)
    x = torch.randn(N, H, W, C, generator=g, device="cuda").to(dtype)
    col, Ho, Wo = run(nv.plan("mr_im2col_nhwc", T, C, Kp), lambda: ops.im2col(x, kh, kw, ph, pw, Kp))
    K = kh * kw * C
    ref = F.unfold(x.double().permute(0, 3, 1, 2), (kh, kw), padding=(ph, pw))
    ref = ref.view(N, C, kh * kw, Ho * Wo).permute(0, 3, 2, 1).reshape(N * Ho * Wo, K)
    assert torch.equal(col[:, :K].double(), ref) and bool((col[:, K:] == 0).all())
    if C % nv.VN[T] or Kp % nv.VN[T]:
        with pytest.raises(_lib.MegReaderB200Error):
            ops.col2im(torch.zeros(N * Ho * Wo, Kp, dtype=dtype, device="cuda"), N, H, W, C, kh, kw, ph, pw)
        return
    d = torch.randn(N * Ho * Wo, Kp, generator=g, device="cuda").to(dtype)
    dx = run(nv.plan("mr_col2im_nhwc", T, C, Kp), lambda: ops.col2im(d, N, H, W, C, kh, kw, ph, pw))

    def fold(t):
        t = t[:, :K].view(N, Ho * Wo, kh * kw, C).permute(0, 3, 2, 1).reshape(N, C * kh * kw, Ho * Wo)
        return F.fold(t, (H, W), (kh, kw), padding=(ph, pw)).permute(0, 2, 3, 1)
    ref, mag = fold(d.double()), fold(d.double().abs())
    _within(dx, ref, kh * kw * U * mag + (_ulp(ref, dtype) if dtype == BF16 else 0), "col2im")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=str)
def test_layout_conversion(cuda, ops, dtype):
    x = torch.randn(3, 5, 7, 9, generator=_gen(11), device="cuda")
    a = run(nv.plan("mr_nchw_to_nhwc", NAME[dtype]), lambda: ops.nchw_to_nhwc(x, 8, dtype))
    assert torch.equal(a[..., :5], x.permute(0, 2, 3, 1).to(dtype)) and bool((a[..., 5:] == 0).all())
    back = run(nv.plan("mr_nhwc_to_nchw", NAME[dtype]), lambda: ops.nhwc_to_nchw(a, 5))
    assert torch.equal(back, x.to(dtype).float())


# ---------------------------------------------------------------- LSTM cell
def _sig(v):
    return 1 / (1 + torch.exp(-v))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,ndir,prev,H,B", LSTM_CASES, ids=str)
def test_lstm_cell(cuda, ops, dtype, ndir, prev, H, B):
    """gate order (i, f, g, o); h lands at row stride ldh = 2H (direction d in columns d*H ..), like the bidirectional
    layer's output.  fp32 uses tanhf / expf, bf16 the tanh.approx activations (about 2^-11 relative)."""
    T = NAME[dtype]
    g = _gen(H + B + ndir)
    tol = 1e-5 if dtype == F32 else 2e-3
    gates = [(torch.randn(B, 4 * H, generator=g, device="cuda") * 2).to(dtype) for _ in range(ndir)]
    gates0 = [t.clone() for t in gates]
    b_ih = [torch.randn(4 * H, generator=g, device="cuda") * 0.3 for _ in range(ndir)]
    b_hh = [torch.randn(4 * H, generator=g, device="cuda") * 0.3 for _ in range(ndir)]
    c_prev = [torch.randn(B, H, generator=g, device="cuda") if prev else None for _ in range(ndir)]
    c_out = [torch.empty(B, H, device="cuda") for _ in range(ndir)]
    out = torch.full((B, 2 * H), 7.0, device="cuda").to(dtype)
    h_out = [out[:, d * H:(d + 1) * H] for d in range(ndir)]
    h_state = [torch.empty(B, H, device="cuda").to(dtype) for _ in range(ndir)]
    run(nv.plan("mr_lstm_cell_fwd", T),
        lambda: ops.lstm_cell_fwd(gates, b_ih, b_hh, c_prev, c_out, h_out, 2 * H, h_state))
    for d in range(ndir):
        pre = gates0[d].double() + b_ih[d].double() + b_hh[d].double()
        i, f, gg, o = _sig(pre[:, :H]), _sig(pre[:, H:2 * H]), torch.tanh(pre[:, 2 * H:3 * H]), _sig(pre[:, 3 * H:])
        c = f * (c_prev[d].double() if prev else 0) + i * gg
        h = o * torch.tanh(c)
        act = torch.cat([i, f, gg, o], 1)
        rnd = 0 if dtype == F32 else 2.0 ** -8
        _within(gates[d], act, (tol + rnd) * act.abs() + tol, "activated gates, direction %d" % d)
        _within(c_out[d], c, tol * (c.abs() + (c_prev[d].double().abs() if prev else 0) + 1), "c, direction %d" % d)
        _within(h_out[d], h, (tol + rnd) * h.abs() + tol, "h, direction %d" % d)
        assert torch.equal(h_state[d], h_out[d])
    if ndir == 1:
        assert bool((out[:, H:] == 7).all()), "the second direction's columns were written"

    # backward from the stored (rounded) activated gates and c
    dh_out = torch.randn(B, 2 * H, generator=g, device="cuda").to(dtype)
    dh_rec = [torch.randn(B, H, generator=g, device="cuda").to(dtype) if prev else None for _ in range(ndir)]
    dc = [torch.randn(B, H, generator=g, device="cuda") for _ in range(ndir)]
    dc0 = [t.clone() for t in dc]
    dgates = [torch.empty(B, 4 * H, device="cuda").to(dtype) for _ in range(ndir)]
    run(nv.plan("mr_lstm_cell_bwd", T),
        lambda: ops.lstm_cell_bwd(gates, c_out, c_prev, [dh_out[:, d * H:(d + 1) * H] for d in range(ndir)], 2 * H,
                                  dh_rec, dc, dgates))
    for d in range(ndir):
        a = gates[d].double()
        i, f, gg, o = a[:, :H], a[:, H:2 * H], a[:, 2 * H:3 * H], a[:, 3 * H:]
        dh = dh_out[:, d * H:(d + 1) * H].double() + (dh_rec[d].double() if prev else 0)
        tc = torch.tanh(c_out[d].double())
        dct = dc0[d].double() + dh * o * (1 - tc * tc)
        cp = c_prev[d].double() if prev else torch.zeros_like(dct)
        want = torch.cat([dct * gg * i * (1 - i), dct * cp * f * (1 - f), dct * i * (1 - gg * gg),
                          dh * tc * o * (1 - o)], 1)
        mag = torch.cat([dct.abs() + dh.abs()] * 4, 1)
        rnd = 0 if dtype == F32 else 2.0 ** -8
        _within(dgates[d], want, tol * mag + rnd * want.abs() + 1e-30, "dgates, direction %d" % d)
        _within(dc[d], dct * f, tol * (dc0[d].double().abs() + dh.abs()) + 1e-30, "dc_prev, direction %d" % d)


# ---------------------------------------------------------------- the engine's BatchNorm buffers, fp32 mode
@pytest.mark.gpu
@pytest.mark.parametrize("momentum", [0.1, None], ids=["momentum0.1", "cumulative"])
def test_engine_running_stats_vs_float64(cuda, momentum):
    """Three training forwards of the CRNN backbone through the engine (fp32) keep every BatchNorm's running_mean,
    running_var and num_batches_tracked equal to the same cnn Sequential run in float64 (momentum=None: the cumulative
    average, factor 1 / num_batches_tracked)."""
    import megreader_b200
    from megreader_b200 import crnn_engine
    from tests.weights import fill_state_dict
    megreader_b200.install_reference_api()
    import backbones
    crnn_engine.set_compute_dtype(F32)
    bb = fill_state_dict(backbones.crnn_backbone(), "bb.").to(cuda).train()
    bns = [m for m in bb.cnn.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    assert len(bns) == 3
    for m in bns:
        m.momentum = momentum
    ref = copy.deepcopy(bb.cnn).double().train()
    g = _gen(21)
    for step in range(3):
        x = torch.randn(4, 3, 32, 100, generator=g, device="cuda") + 0.5 * step
        feat = bb(x)
        with torch.no_grad():
            ref(x.double())
        feat.float().sum().backward()
    for m, r in zip(bns, [m for m in ref.modules() if isinstance(m, torch.nn.BatchNorm2d)]):
        assert int(m.num_batches_tracked) == int(r.num_batches_tracked) == 3
        sd = r.running_var.sqrt()
        _within(m.running_mean, r.running_mean, 1e-4 * (r.running_mean.abs() + sd), "running_mean")
        _within(m.running_var, r.running_var, 1e-4 * r.running_var.abs() + 1e-6, "running_var")
