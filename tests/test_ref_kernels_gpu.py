"""GPU parity, kernel against kernel: the product's sm_90a kernels (through the C-ABI) versus the reference's OWN CUDA ops --
the UNMODIFIED sources under ops/ctc_2d/csrc and assets/ops/dcn/src, compiled by oracle/build_ref.py into oracle/_ref/*.so
(SURVEY.md section 8c's "third check").  What those kernels returned for every case is stored under tests/golden/refk_*.npz
(oracle/make_ref_golden.py ran them on an H100; arrays above 512 elements as a fixed seeded sample of mostly non-zero entries, tests.cases.sample_indices), so the comparison runs on
any checkout; where oracle/_ref is built the reference kernels also run live and every element is compared.  This is the pin
for every native op of the path: 2D-CTC K1/K2/K3 in fp32 and fp64 incl. the realistic (saturating-python) cfg-3 regime,
DCNv1/v2 incl. the offset-size != output-size quirk, and deformable PS-RoI pooling (row A13, previously unpinned).
The same inputs also go through the CPU restatements in oracle/*.c, so the oracle itself is pinned to the reference here."""
import numpy as np
import pytest
import torch

import os

from oracle import build_ref, capi
from tests.cases import ctc2d_case
from tests.deform_pool_cases import CASES as POOL_CASES, make as pool_make

pytestmark = pytest.mark.gpu


GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _references(op, case_id, names, run_live, share=None):
    """[(reference outputs by name, select)]: the stored sample of what the reference kernels returned, and, where oracle/_ref
    is built, their live outputs in full.  select(array, name) cuts one of our arrays down to the elements the reference entry
    `name` holds.  run_live(module) -> tuple of tensors in the order of `names`.  share = {name: other}: the stored sample of `name`
    was taken at the indices of `other` (arrays that are compared element against element)."""
    with np.load(os.path.join(GOLD, "refk_%s.npz" % op)) as g:
        stored = {n: g["%s.%s" % (case_id, n)] for n in names}
        idx = {n: g["%s.%s__idx" % (case_id, n)] for n in names if "%s.%s__idx" % (case_id, n) in g.files}

    def pick(a, n):
        a = np.asarray(a).reshape(-1)
        return a[idx[n]] if n in idx else a
    refs = [(stored, pick)]
    mod = build_ref.load("ref_" + op)
    if mod is not None:
        live = run_live(mod)
        torch.cuda.synchronize()
        refs.append(({n: t.cpu().numpy().reshape(-1) for n, t in zip(names, live)}, lambda a, n: np.asarray(a).reshape(-1)))
    return refs


def _dev(cuda, *arrs):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(cuda) for a in arrs]


# ------------------------------------------------------------------------------------------------ 2D-CTC
CTC_CASES = [
    # seed, T, H, N, C, S, Lmax, ragged, peak
    (31, 32, 8, 64, 38, 32, 12, False, 0.0),    # cfg-3 shape, random logits: loss ~ 90-130 (python reference saturates here)
    (32, 32, 8, 33, 38, 32, 16, True, 0.0),     # ragged input lengths, longest targets
    (33, 32, 8, 16, 38, 32, 12, False, 6.0),    # peaked (trained-model-like) regime
    (34, 16, 4, 9, 11, 8, 6, True, 0.0),
    (35, 64, 1, 5, 38, 32, 20, False, 0.0),     # H = 1 (1D CTC through the 2D op)
    (36, 8, 3, 3, 4001, 4, 4, False, 0.0),      # large alphabet
    (37, 32, 8, 2048, 38, 32, 12, False, 0.0),  # the CRNN-2D head's batch
    (38, 32, 8, 6, 5000, 32, 32, True, 0.0),    # ChineseCharset-sized alphabet at the real T / H, targets up to 32 labels
    (39, 32, 8, 11, 38, 32, 32, False, 0.0),    # longest targets (65 states: 3 states per lane, slot rounds)
]


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", CTC_CASES, ids=[str(c[0]) for c in CTC_CASES])
def test_ctc2d_vs_reference_kernels(cuda, case, dtype):
    """ops/ctc_2d/csrc/cuda/ctc2d_cuda_kernel.cu K1 (:54-211), K2 (:254-368), K3 (:427-517) run on this GPU.  T divides 1024
    in every case, so the reference's K3 aliasing race (SURVEY App. B1.5) is not in play and its output is deterministic."""
    from megreader_b200 import ctc2d
    seed, T, H, N, C, S, Lmax, ragged, peak = case
    if dtype == np.float64 and N > 256:
        pytest.skip("fp64 at the large batch adds nothing")
    if dtype == np.float64 and C > 1024:
        pytest.skip("fp64 with a >1k-class alphabet: the fp64 DP keeps [T, C] rows on chip -> MR_ERR_UNSUPPORTED (DESIGN.md section 7)")
    assert 1024 % T == 0
    lp, tg, il, tl = ctc2d_case(seed, T, H, N, C, S, Lmax, peak=peak, ragged_T=ragged, dtype=dtype)
    go = (1.0 / tl).astype(dtype)
    d_lp, d_tg, d_il, d_tl, d_go = _dev(cuda, lp, tg, il, tl, go)

    def run_ctc_ref(ref):
        r_nll, r_la = ref.ctc2d_forward(d_lp, d_tg, d_il, d_tl, 0, 0.0)
        return r_nll, r_la, ref.ctc2d_backward(d_go, d_lp, d_tg, d_il, d_tl, r_nll, r_la, 0)
    refs = _references("ctc2d", "%d-%s" % (seed, np.dtype(dtype).name), ("nll", "log_alpha", "grad"), run_ctc_ref)
    nll, la = ctc2d.ctc2d_forward(d_lp, d_tg, d_il, d_tl, 0, 0.0)
    gr = ctc2d.ctc2d_backward(d_go, d_lp, d_tg, d_il, d_tl, nll, la, 0)
    rt = 1e-4 if dtype == np.float32 else 1e-9
    nll, la, gr = [t.cpu().numpy() for t in (nll, la, gr)]
    loss = x = None
    if dtype == np.float32:   # training pair (what ops.ctc_loss_2d runs when log_probs requires grad): same values
        x = d_lp.clone().requires_grad_(True)
        loss = ctc2d.ctc_loss_2d(x, d_tg, d_il, d_tl)
        (loss * d_go).sum().backward()
    o_nll = o_gr = None
    if N <= 64 and C <= 64:   # the CPU restatement is pinned to the same reference output (small cases: the C oracle is serial)
        o_nll, o_la = capi.ctc2d_forward(lp.astype(np.float64), tg, il, tl)
        o_gr = capi.ctc2d_backward(go.astype(np.float64), lp.astype(np.float64), tg, il, tl, o_nll, o_la)
    for r, sel in refs:
        r_nll, r_la, r_gr = r["nll"], r["log_alpha"], r["grad"]
        assert np.isfinite(r_nll).all()
        np.testing.assert_allclose(sel(nll, "nll"), r_nll, rtol=rt)
        fin = np.isfinite(r_la)
        assert np.array_equal(np.isfinite(sel(la, "log_alpha")), fin), "log_alpha -inf pattern differs from the reference kernel"
        np.testing.assert_allclose(sel(la, "log_alpha")[fin], r_la[fin], rtol=rt, atol=1e-4 if dtype == np.float32 else 1e-9)
        assert np.array_equal(sel(gr, "grad") == 0, r_gr == 0), "zero pattern of the gradient differs from the reference K3"
        np.testing.assert_allclose(sel(gr, "grad"), r_gr, rtol=2e-4 if dtype == np.float32 else 1e-8, atol=2e-5 if dtype == np.float32 else 1e-10)
        if loss is not None:
            np.testing.assert_allclose(sel(loss.detach().cpu().numpy(), "nll"), r_nll, rtol=rt)
            np.testing.assert_allclose(sel(x.grad.cpu().numpy(), "grad"), r_gr, rtol=2e-4, atol=2e-5)
        if o_nll is not None:
            np.testing.assert_allclose(sel(o_nll, "nll"), r_nll, rtol=rt)
            np.testing.assert_allclose(sel(o_gr, "grad"), r_gr, rtol=2e-4 if dtype == np.float32 else 1e-8,
                                       atol=2e-5 if dtype == np.float32 else 1e-10)


# ------------------------------------------------------------------------------------------------ DCN v1 / v2
def _dcn_inputs(seed, B, C, H, W, Cout, k, s, p, d, group, dg, big_offset):
    rng = np.random.RandomState(seed)
    Ho = (H + 2 * p - (d * (k - 1) + 1)) // s + 1
    Wo = (W + 2 * p - (d * (k - 1) + 1)) // s + 1
    oh, ow = (H, W) if big_offset else (Ho, Wo)
    x = rng.standard_normal((B, C, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, C // group, k, k)) / np.sqrt(C * k * k)).astype(np.float32)
    b = rng.standard_normal((Cout,)).astype(np.float32)
    off = (rng.standard_normal((B, 2 * k * k * dg, oh, ow)) * 1.5).astype(np.float32)
    m = (1 / (1 + np.exp(-rng.standard_normal((B, k * k * dg, oh, ow))))).astype(np.float32)
    go = rng.standard_normal((B, Cout, Ho, Wo)).astype(np.float32)
    return x, w, b, off, m, go, Ho, Wo


DCN_CASES = [
    # B, C, H, W, Cout, k, s, p, d, group, dg, with_bias, big_offset
    (2, 8, 9, 11, 8, 3, 1, 1, 1, 1, 1, True, False),
    (3, 8, 8, 8, 8, 3, 2, 1, 1, 1, 1, False, True),       # stride 2 with INPUT-sized offset/mask maps (SURVEY App. B2.1)
    (2, 16, 10, 7, 8, 3, 1, 2, 2, 2, 2, True, False),     # dilation 2, groups, deformable groups
    (4, 128, 16, 16, 128, 3, 1, 1, 1, 1, 1, False, False),
    (2, 256, 16, 16, 256, 3, 2, 1, 1, 1, 1, False, True),  # layer-3 first block geometry (stride 2, big offset)
    (2, 64, 12, 20, 64, 3, 1, 1, 1, 1, 1, True, False),
    (2, 128, 13, 19, 256, 3, 1, 1, 1, 1, 1, True, False),  # fused backward, ragged 8 x 16 tiles, Cout = 2 x 128
]


def _close(a, ref, name, sel, tol=1e-4, what=None):
    a = sel(a.cpu().numpy(), name)
    scale = max(1.0, float(np.abs(ref).max()))
    np.testing.assert_allclose(a, ref, rtol=tol, atol=tol * scale, err_msg=what or name)


@pytest.mark.parametrize("case", DCN_CASES, ids=[str(i) for i in range(len(DCN_CASES))])
def test_dcnv2_vs_reference_kernels(cuda, case):
    """assets/ops/dcn/src/deform_conv_cuda.cpp:486-679 + deform_conv_cuda_kernel.cu:569-766 run on this GPU."""
    from megreader_b200 import dcn
    B, C, H, W, Cout, k, s, p, d, group, dg, with_bias, big = case
    x, w, b, off, m, go, Ho, Wo = _dcn_inputs(11, B, C, H, W, Cout, k, s, p, d, group, dg, big)
    tx, tw, tb, toff, tm, tgo = _dev(cuda, x, w, b, off, m, go)
    e = lambda: tx.new_empty(0)  # noqa: E731

    def run_dcn_ref(ref):
        r_out = tx.new_empty(B, Cout, Ho, Wo)
        ref.modulated_deform_conv_cuda_forward(tx, tw, tb, e(), toff, tm, r_out, e(), k, k, s, s, p, p, d, d, group, dg, with_bias)
        r_gi, r_gw, r_gb, r_goff, r_gm = [torch.zeros_like(t) for t in (tx, tw, tb, toff, tm)]
        ref.modulated_deform_conv_cuda_backward(tx, tw, tb, e(), toff, tm, e(), r_gi, r_gw, r_gb, r_goff, r_gm, tgo, k, k, s, s,
                                                p, p, d, d, group, dg, with_bias)
        return r_out, r_gi, r_gw, r_gb, r_goff, r_gm
    names = ("output", "grad_input", "grad_weight", "grad_bias", "grad_offset", "grad_mask")
    refs = _references("deform_conv", "v2-%d" % DCN_CASES.index(case), names, run_dcn_ref)
    out = tx.new_empty(B, Cout, Ho, Wo)
    dcn.modulated_deform_conv_cuda_forward(tx, tw, tb, None, toff, tm, out, None, k, k, s, s, p, p, d, d, group, dg, with_bias)
    gi, gw, gb, goff, gm = [torch.zeros_like(t) for t in (tx, tw, tb, toff, tm)]
    dcn.modulated_deform_conv_cuda_backward(tx, tw, tb, None, toff, tm, None, gi, gw, gb, goff, gm, tgo, k, k, s, s, p, p, d, d,
                                            group, dg, with_bias)
    for r, sel in refs:
        for n, mine in zip(names, (out, gi, gw, gb, goff, gm)):
            if n != "grad_bias" or with_bias:
                _close(mine, r[n], n, sel)
    if big:   # the tail of each [., Hi, Wi] slab stays zero (flat (Ho,Wo) indexing), as in the reference
        assert float(goff.view(B, -1)[:, 2 * k * k * dg * Ho * Wo:].abs().max()) == 0.0


DCNV1_CASES = [(4, 8, 9, 11, 8, 3, 1, 1, 1, 1, 1), (4, 16, 12, 12, 8, 3, 2, 1, 1, 2, 2), (2, 64, 16, 16, 64, 3, 1, 1, 1, 1, 1)]


@pytest.mark.parametrize("case", DCNV1_CASES, ids=["a", "b", "c"])
def test_dcnv1_vs_reference_kernels(cuda, case):
    """deform_conv_{forward,backward_input,backward_parameters}_cuda, deform_conv_cuda.cpp:151-484 (K5-K7)."""
    from megreader_b200 import dcn
    B, C, H, W, Cout, k, s, p, d, group, dg = case
    x, w, _, off, _, go, Ho, Wo = _dcn_inputs(12, B, C, H, W, Cout, k, s, p, d, group, dg, False)
    tx, tw, toff, tgo = _dev(cuda, x, w, off, go)
    e = lambda: tx.new_empty(0)  # noqa: E731
    # im2col_step = B, as functions/deform_conv.py:43 picks for B <= 64.  (The reference's forward re-views `columns` inside
    # its batch loop, deform_conv_cuda.cpp:225, so more than one loop iteration cannot work at all.)
    step = B

    def run_v1_ref(ref):
        r_out = tx.new_empty(B, Cout, Ho, Wo)
        ref.deform_conv_forward_cuda(tx, tw, toff, r_out, e(), e(), k, k, s, s, p, p, d, d, group, dg, step)
        r_gi, r_goff, r_gw = torch.zeros_like(tx), torch.zeros_like(toff), torch.zeros_like(tw)
        ref.deform_conv_backward_input_cuda(tx, toff, tgo, r_gi, r_goff, tw, e(), k, k, s, s, p, p, d, d, group, dg, step)
        # backward_parameters does zeros_like(transposed view).view(...) (deform_conv_cuda.cpp:423-430), which only works with
        # today's stride-preserving zeros_like when the transposed dimension has size 1: one sample per call, accumulating
        # into gradWeight exactly as the op is specified to do
        for b in range(B):
            ref.deform_conv_backward_parameters_cuda(tx[b:b + 1], toff[b:b + 1], tgo[b:b + 1], r_gw, e(), e(), k, k, s, s, p, p, d, d,
                                                     group, dg, 1.0, 1)
        return r_out, r_gi, r_goff, r_gw
    names = ("output", "grad_input", "grad_offset", "grad_weight")
    refs = _references("deform_conv", "v1-%d-%d" % (C, Cout), names, run_v1_ref)
    txg, toffg, twg = [t.clone().requires_grad_(True) for t in (tx, toff, tw)]
    out = dcn.deform_conv(txg, toffg, twg, s, p, d, group, dg)
    out.backward(tgo)
    for r, sel in refs:
        for n, mine in zip(names, (out.detach(), txg.grad, toffg.grad, twg.grad)):
            _close(mine, r[n], n, sel)


# ------------------------------------------------------------------------------------------------ deformable PS-RoI pooling
@pytest.mark.parametrize("name", sorted(POOL_CASES))
def test_deform_pool_vs_reference_kernels(cuda, name):
    """assets/ops/dcn/src/deform_pool_cuda_kernel.cu:52-263 (K11/K12) run on this GPU: pins row A13 and, through the same
    inputs, oracle/deform_pool_oracle.c."""
    from megreader_b200 import deform_pool as dp
    data, rois, trans, a = pool_make(name)
    d, r = _dev(cuda, data.astype(np.float32), rois.astype(np.float32))
    t = _dev(cuda, trans.astype(np.float32))[0] if trans is not None else d.new_empty(0)
    n, od, P = rois.shape[0], a["output_dim"], a["pooled"]
    args = (int(a["no_trans"]), float(a["spatial_scale"]), od, a["group_size"], P, a["part_size"], a["sample_per_part"],
            float(a["trans_std"]))
    rng = np.random.RandomState(1)
    go = torch.from_numpy(rng.standard_normal((n, od, P, P)).astype(np.float32)).to(cuda)

    def run_pool_ref(ref):
        r_out, r_cnt = d.new_zeros(n, od, P, P), d.new_zeros(n, od, P, P)
        ref.deform_psroi_pooling_cuda_forward(d, r, t, r_out, r_cnt, *args)
        r_gin, r_gtr = torch.zeros_like(d), torch.zeros_like(t)
        ref.deform_psroi_pooling_cuda_backward(go, d, r, t, r_cnt, r_gin, r_gtr, *args)
        return r_out, r_cnt, r_gin, r_gtr
    refs = _references("deform_pool", name, ("out", "top_count", "input_grad", "trans_grad"), run_pool_ref, share={"top_count": "out"})
    out, cnt = d.new_zeros(n, od, P, P), d.new_zeros(n, od, P, P)
    dp.deform_psroi_pooling_cuda_forward(d, r, t, out, cnt, *args)
    gin, gtr = torch.zeros_like(d), torch.zeros_like(t)
    dp.deform_psroi_pooling_cuda_backward(go, d, r, t, cnt, gin, gtr, *args)
    o_out, o_cnt = capi.deform_psroi_forward(data, rois, trans, **a)
    for ref_, sel in refs:
        # same fp32 arithmetic on both sides: the sample counts must agree exactly, values to rounding
        assert np.array_equal(sel(cnt.cpu().numpy(), "top_count"), ref_["top_count"]), "top_count differs from the reference kernel"
        _close(out, ref_["out"], "out", sel, 1e-5)
        _close(gin, ref_["input_grad"], "input_grad", sel, 1e-4, "input_grad (atomic order differs)")
        if trans is not None:
            _close(gtr, ref_["trans_grad"], "trans_grad", sel, 1e-4)
        # the fp64 CPU restatement against the reference kernel (bins whose samples sit on a half-pixel border within fp32
        # rounding may count differently in fp64: they must be rare, and everything else must agree)
        same = sel(o_cnt, "top_count") == ref_["top_count"]
        assert same.mean() > 0.98
        np.testing.assert_allclose(sel(o_out, "out")[same], ref_["out"][same], rtol=1e-4, atol=1e-4)
