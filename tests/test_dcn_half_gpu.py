"""GPU: deformable convolution in float16 / bfloat16 (the half-precision fused wgmma kernels of csrc/dcn_tcgen05.cu and the
fp32 fallback outside the fused path) against the float64 oracle (oracle/dcn_oracle.c) on the same T-rounded inputs.

Error bound, element-wise, with u the unit roundoff of T (2^-8 bf16, 2^-11 fp16) and u_w = u for float32 weights (they are
packed to T), 0 for T weights (the oracle gets the same T values):
  output       (u + u_w + 2^-16) * sum |W| |col|  +  u |ref|
               each column value (bilinear blend x mask, fp32) is rounded once to T, the weight once to T, the K sum is fp32
               (2^-16 leaves ~100x margin over an fp32 sum, as in wgmma_variants.bound), the stored output is rounded once.
               sum |W| |col| is the oracle's forward on |x|, |W|, |bias|, |mask| (the bilinear weights are >= 0).
  grad_weight  (u + 2^-16) * sum |go| |col|  +  u_store |ref|      (go is already T; fp32 atomics; u_store = u for T weights)
  grad_input   (u_w + 2^-16) * sum |W| |go| m w_bilinear  +  u |ref|     (Wᵀ go in fp32 from T operands, fp32 scatter)
  grad_mask    (u_w + 2^-16) * sum_c |Wᵀ go|_c blend(|x|)  +  u |ref|
  grad_offset  (u_w + 2^-16) * 4 max|x| * m * sum_c sum_co |W| |go|  +  u |ref|
               (|d blend / d position| <= sum of the four valid corner magnitudes <= 4 max|x|)
  grad_bias    2^-16 * sum |go|  +  u_store |ref|
The magnitudes of grad_weight / grad_input / grad_mask are the oracle's backward on absolute values.
"""
import numpy as np
import pytest
import torch

from oracle import capi
from tests import wgmma_variants as wv
from tests.test_dcn_gpu import CASES, _inputs

pytestmark = pytest.mark.gpu

U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
DTYPES = [torch.float16, torch.bfloat16]
ACC = 2.0 ** -16

BIG_OFFSET_CASE = (2, 128, 13, 19, 128, 3, 2, 1, 1, 1, 1, True, True)   # stride 2 with input-sized offsets (App. B2.1)
FULL_TILE_CASE = (2, 128, 16, 32, 128, 3, 1, 1, 1, 1, 1, True, True)    # every 8 x 16 tile full: the last tile row is checked
FUSED = [("stride2_ragged", CASES[9], False), ("c256", CASES[10], False), ("v1_dil2", CASES[11], False),
         ("c64_fwd_fused", CASES[8], False), ("big_offset", BIG_OFFSET_CASE, True),
         ("full_tiles", FULL_TILE_CASE, False)]
FALLBACK = [("c4", CASES[0], False), ("grouped_dg2", CASES[2], False), ("dg3", CASES[3], False)]

HALF_VARIANTS = frozenset("dcn_%s_half_kernel<%s>" % (k, t) for k in ("fwd", "wgrad", "dgrad")
                          for t in ("__half", "__nv_bfloat16"))
_TNAME = {torch.float16: "__half", torch.bfloat16: "__nv_bfloat16"}


def _run(cuda, case, dt, wdt, big, seed=1):
    """-> (T inputs as float64 numpy, our outputs / gradients as float64 numpy)."""
    from megreader_b200 import dcn
    B, C, H, W, Cout, k, s, p, d, group, dg, modulated, with_bias = case
    x, w, b, off, m, go = _inputs(seed, B, C, H, W, Cout, k, s, p, d, group, dg, big_offset=big)
    tx, toff, tm = [torch.from_numpy(a).to(cuda, dt).requires_grad_(True) for a in (x, off, m)]
    tw, tb = [torch.from_numpy(a).to(cuda, wdt).requires_grad_(True) for a in (w, b)]
    tgo = torch.from_numpy(go).to(cuda, dt)
    if modulated:
        out = dcn.modulated_deform_conv(tx, toff, tm, tw, tb if with_bias else None, s, p, d, group, dg)
    else:
        out = dcn.deform_conv(tx, toff, tw, s, p, d, group, dg)
    out.backward(tgo)
    f = lambda t: t.detach().double().cpu().numpy()  # noqa: E731
    inp = dict(x=f(tx), w=f(tw), b=f(tb) if with_bias else None, off=f(toff), m=f(tm) if modulated else None, go=f(tgo))
    got = dict(out=out, gi=tx.grad, gw=tw.grad, goff=toff.grad, gm=tm.grad if modulated else None,
               gb=tb.grad if with_bias else None)
    return inp, got


def _check_case(cuda, case, dt, wdt, big):
    B, C, H, W, Cout, k, s, p, d, group, dg, modulated, with_bias = case
    inp, got = _run(cuda, case, dt, wdt, big)
    assert got["out"].dtype == dt and got["gi"].dtype == dt and got["goff"].dtype == dt
    assert got["gw"].dtype == wdt and (got["gb"] is None or got["gb"].dtype == wdt)
    x, w, b, off, m, go = inp["x"], inp["w"], inp["b"], inp["off"], inp["m"], inp["go"]
    geo = (s, p, d, group, dg)
    o_ref = capi.dcn_forward(x, w, b, off, m, *geo)
    gi, gw, gb, goff, gm = capi.dcn_backward(x, w, b, off, m, go, *geo)
    ax, aw, am, ago = np.abs(x), np.abs(w), None if m is None else np.abs(m), np.abs(go)
    o_abs = capi.dcn_forward(ax, aw, None if b is None else np.abs(b), off, am, *geo)
    gi_abs, gw_abs, _, _, gm_abs = capi.dcn_backward(ax, aw, None, off, am, ago, *geo)
    u = U[dt]
    u_w = u if wdt == torch.float32 else 0.0
    u_store = u if wdt != torch.float32 else 0.0
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    bounds = {
        "out": (u + u_w + ACC) * o_abs + u * np.abs(o_ref),
        "gi": (u_w + ACC) * gi_abs + u * np.abs(gi),
        "gw": (u + ACC) * gw_abs + u_store * np.abs(gw),
    }
    refs = {"out": o_ref, "gi": gi, "gw": gw, "goff": goff}
    # grad_offset: flat (Ho, Wo) layout inside each sample slab of the offset tensor
    K, Ho, Wo = k * k, o_ref.shape[2], o_ref.shape[3]
    P = Ho * Wo
    colsum = aw.sum(axis=1).reshape(Cout, K)                                 # sum_c |W[co, c, k]|
    S = np.einsum("ok,bop->bkp", colsum, ago.reshape(B, Cout, P))            # sum_c sum_co |W| |go|
    mflat = np.ones((B, dg * K, P)) if m is None else am.reshape(B, -1)[:, :dg * K * P].reshape(B, dg * K, P)
    xmax = ax.reshape(B, -1).max(axis=1)[:, None, None]
    mag = 4 * xmax * np.tile(S, (1, dg, 1)) * mflat                         # [B][dg*K][P], per mask channel
    goff_mag = np.zeros_like(goff).reshape(B, -1)
    goff_mag[:, :2 * dg * K * P] = np.repeat(mag, 2, axis=1).reshape(B, -1)
    bounds["goff"] = (u_w + ACC) * goff_mag.reshape(goff.shape) + u * np.abs(goff)
    if m is not None:
        refs["gm"] = gm
        bounds["gm"] = (u_w + ACC) * gm_abs + u * np.abs(gm)
    if with_bias:
        refs["gb"] = gb
        bounds["gb"] = ACC * ago.sum(axis=(0, 2, 3)) + u_store * np.abs(gb)
    for key in refs:
        wv.assert_within(got[key].detach().double().cpu(), T(refs[key]), T(bounds[key]), "%s %s" % (dt, key))


@pytest.mark.parametrize("wdt", ["T", "f32"])
@pytest.mark.parametrize("dt", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("name,case,big", FUSED + FALLBACK, ids=[c[0] for c in FUSED + FALLBACK])
def test_dcn_half_vs_oracle(cuda, name, case, big, dt, wdt):
    _check_case(cuda, case, dt, dt if wdt == "T" else torch.float32, big)


def _fused_variants(dt, backward_data):
    t = _TNAME[dt]
    names = {"dcn_fwd_half_kernel<%s>" % t, "dcn_wgrad_half_kernel<%s>" % t}
    if backward_data:
        names.add("dcn_dgrad_half_kernel<%s>" % t)
    return names


# (case, big offsets, the half kernels forward + backward launch); C = 64 has no fused data gradient, so its backward runs
# the fp32 fallback and only the forward is fused
PATH_CASES = [(CASES[9], False, True), (CASES[11], False, True), (BIG_OFFSET_CASE, True, True)]
VARIANTS = set()
for _dt in DTYPES:
    VARIANTS |= _fused_variants(_dt, True)


@pytest.mark.parametrize("dt", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("idx", range(len(PATH_CASES)))
def test_dcn_half_path(cuda, dt, idx):
    """torch.profiler: the half kernels ran, and no fp32 fused or unfused DCN kernel.  A trace without any DCN kernel
    record only warns (the rule of wgmma_variants.run_variant)."""
    import warnings
    case, big, data = PATH_CASES[idx]
    _, names = wv.launched_kernels(lambda: _run(cuda, case, dt, dt, big))
    dcn_names = {n for n in names if n.startswith("dcn_")}
    if not dcn_names:
        warnings.warn("torch.profiler recorded no DCN kernel: path not checked (saw %s)" % sorted(names))
        return
    want = _fused_variants(dt, data)
    assert want <= dcn_names, "expected %s, the profiler saw %s" % (sorted(want), sorted(dcn_names))
    fp32 = {n for n in dcn_names if "tcgen05" in n or n in ("dcn_im2col_kernel", "dcn_col2im_kernel")}
    assert not fp32, "fp32 DCN kernels ran on the half path: %s" % sorted(fp32)


def test_dcn_half_c64_backward_falls_back(cuda):
    """C % 128 != 0: the fused half forward, then the fp32 fallback for the backward (the data gradient needs C % 128 == 0)."""
    _, names = wv.launched_kernels(lambda: _run(cuda, CASES[8], torch.float16, torch.float16, False))
    if not any(n.startswith("dcn_") for n in names):
        pytest.skip("torch.profiler recorded no DCN kernel")
    assert "dcn_fwd_half_kernel<__half>" in names
    assert "dcn_dgrad_half_kernel<__half>" not in names and "dcn_col2im_kernel" in names


# ---- autocast ------------------------------------------------------------------------------------------------------
def _pack(cls, cuda, C, seed):
    torch.manual_seed(seed)
    mod = cls(C, C, 3, stride=1, padding=1).to(cuda)
    off_conv = mod.conv_offset_mask if hasattr(mod, "conv_offset_mask") else mod.conv_offset
    with torch.no_grad():
        off_conv.weight.normal_(0, 0.02)
        off_conv.bias.normal_(0, 0.3)
    return mod, off_conv


@pytest.mark.parametrize("dt", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("modulated", [True, False], ids=["v2", "v1"])
def test_dcn_autocast_pack_modules(cuda, dt, modulated):
    """Under torch.autocast the offset conv returns T for an fp32 input: the op upcasts the offsets and runs in fp32
    (output fp32, weight.grad fp32).  A T input (a half-precision trunk) with the same fp32 module runs the half kernels:
    output T, weight.grad fp32.  Output, weight.grad and the op's input gradient are checked against the fp32 op on the same
    rounded input / offsets / mask, within the bounds of the module docstring (fp32 weights: u_w = u) plus 1e-4 of the
    magnitude for the fp32 reference's own error (its hi / lo bf16 split).  The module's x.grad also holds the offset conv's
    share, so the input gradient is taken from the op called the way the module calls it."""
    from megreader_b200 import dcn
    cls = dcn.ModulatedDeformConvPack if modulated else dcn.DeformConvPack
    mod, off_conv = _pack(cls, cuda, 128, 3)
    x = torch.randn(2, 128, 12, 20, device=cuda)
    W, bias = mod.weight.detach(), mod.bias.detach() if modulated else None

    def op(xx, offs, mk, w, b):
        return dcn.modulated_deform_conv(xx, offs, mk, w, b, 1, 1, 1) if modulated else dcn.deform_conv(xx, offs, w, 1, 1, 1)

    def fp32_op(xx, offs, mk, w, b, go):
        """(output, grad of x, grad of w) of the fp32 op"""
        xx, w = xx.clone().requires_grad_(True), w.clone().requires_grad_(True)
        o = op(xx, offs, mk, w, b)
        o.backward(go)
        return o.detach(), xx.grad, w.grad

    for xin, out_dt in ((x, torch.float32), (x.to(dt), dt)):
        mod.zero_grad()
        xi = xin.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=dt):
            out = mod(xi)
            om = off_conv(xi).detach()
        assert out.dtype == out_dt and om.dtype == dt
        go = torch.randn(out.shape, device=cuda).to(out_dt)
        out.backward(go)
        gw = mod.weight.grad.clone()
        assert gw.dtype == torch.float32 and torch.isfinite(gw).all()
        # the offsets / mask exactly as the module hands them to the op (T), and the op's own input gradient
        if modulated:
            o1, o2, mk_t = torch.chunk(om, 3, dim=1)
            offs_t, mk_t = torch.cat((o1, o2), 1), torch.sigmoid(mk_t)
        else:
            offs_t, mk_t = om, None
        xd = xin.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=dt):
            od = op(xd, offs_t, mk_t, mod.weight, mod.bias if modulated else None)
        od.backward(go)
        assert xd.grad.dtype == out_dt
        # fp32 reference on the same rounded values
        offs, mk, xr, gor = offs_t.float(), None if mk_t is None else mk_t.float(), xin.float(), go.float()
        ref, ref_gx, ref_gw = fp32_op(xr, offs, mk, W, bias, gor)
        if out_dt == torch.float32:
            torch.testing.assert_close(out.detach(), ref, rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(xd.grad, ref_gx, rtol=1e-4, atol=1e-4 * float(ref_gx.abs().max()))
            torch.testing.assert_close(gw, ref_gw, rtol=1e-4, atol=1e-4 * float(ref_gw.abs().max()))
            continue
        # magnitudes |W| |col|, |W| |go| m w and |go| |col| from the fp32 op on absolute values
        mag, mag_gx, mag_gw = fp32_op(xr.abs(), offs, mk, W.abs(), None, gor.abs())
        u = U[dt]
        d = lambda t: t.detach().double()  # noqa: E731
        wv.assert_within(d(out), d(ref), d((2 * u + ACC + 1e-4) * mag + u * ref.abs()), "autocast %s output" % dt)
        wv.assert_within(d(xd.grad), d(ref_gx), d((u + ACC + 1e-4) * mag_gx + u * ref_gx.abs()), "autocast %s grad_input" % dt)
        wv.assert_within(d(gw), d(ref_gw), d((u + ACC + 1e-4) * mag_gw), "autocast %s weight.grad" % dt)


# ---- dtype rules -----------------------------------------------------------------------------------------------------
def test_dcn_dtype_rules(cuda):
    """every row of the dtype table of megreader_b200/dcn.py, including the RuntimeError rows"""
    from megreader_b200 import dcn
    B, C, H, W, Cout = 1, 128, 6, 7, 128
    x, w, b, off, m, go = _inputs(4, B, C, H, W, Cout, 3, 1, 1, 1, 1, 1)
    t = lambda a, dt: torch.from_numpy(a).to(cuda, dt).requires_grad_(True)  # noqa: E731
    f32 = torch.float32
    for xd, wd, offd in ((f32, f32, f32), (f32, f32, torch.float16), (torch.float16, torch.float16, torch.float16),
                         (torch.float16, f32, f32), (torch.bfloat16, torch.bfloat16, f32), (torch.bfloat16, f32, torch.bfloat16)):
        tx, tw, tb, toff, tm = t(x, xd), t(w, wd), t(b, wd), t(off, offd), t(m, offd)
        out = dcn.modulated_deform_conv(tx, toff, tm, tw, tb, 1, 1, 1)
        assert out.dtype == xd
        out.backward(torch.from_numpy(go).to(cuda, xd))
        assert tx.grad.dtype == xd and tw.grad.dtype == wd and tb.grad.dtype == wd
        assert toff.grad.dtype == offd and tm.grad.dtype == offd
        for g in (out, tx.grad, tw.grad, tb.grad, toff.grad, tm.grad):
            assert torch.isfinite(g.float()).all()
    bad = ((torch.float64, torch.float64, None), (f32, torch.float16, None), (torch.float16, torch.float64, None),
           (torch.bfloat16, torch.float16, None), (torch.float16, torch.float16, f32), (f32, f32, torch.float16))
    for xd, wd, bd in bad:
        tx, tw, toff, tm = t(x, xd), t(w, wd), t(off, xd), t(m, xd)
        tb = None if bd is None else t(b, bd)
        with pytest.raises(RuntimeError, match="unsupported dtypes"):
            dcn.modulated_deform_conv(tx, toff, tm, tw, tb, 1, 1, 1)
    # contiguity messages are unchanged on the half path
    tx = t(x, torch.float16)
    out = tx.new_empty(B, Cout, H, W)
    with pytest.raises(RuntimeError, match="input tensor has to be contiguous"):
        dcn.modulated_deform_conv_cuda_forward(tx.detach().transpose(2, 3), t(w, torch.float16).detach(), None, None,
                                               t(off, torch.float16).detach(), t(m, torch.float16).detach(), out, None,
                                               3, 3, 1, 1, 1, 1, 1, 1, 1, 1, False)
