"""GPU parity in float16, kernel against kernel: the half-precision DCNv2 path against the reference's OWN fp16 kernels (its four
DCN dispatches are AT_DISPATCH_FLOATING_TYPES_AND_HALF; oracle/_ref/ref_deform_conv.so built by oracle/build_ref.py), both
measured against the float64 oracle (oracle/dcn_oracle.c) on the same fp16 inputs.

The reference computes sampling positions, bilinear weights and column values in half and accumulates grad_input / grad_weight
in half; the half path here computes positions and blend in fp32, rounds each column value once to fp16 and sums in fp32.  So
per array, our relative L2 error against the oracle must not exceed the reference's, or the fp16 rounding floor when that is
larger: 2u = 2^-10, one rounding of the column value plus one of the stored result (u = 2^-11 for fp16).

What the reference kernels returned is stored in tests/golden/refk_deform_conv_f16.npz (a fixed seeded sample of each array,
tests.cases.sample_indices, with its flat indices), so the comparison runs on any checkout; where oracle/_ref is built the
reference also runs live and the whole arrays are compared.  Record the golden on a GPU with oracle/_ref built:

    python -m tests.test_dcn_half_ref_gpu OUT_DIR          # -> OUT_DIR/refk_deform_conv_f16.npz (refk_*.npz are not touched)
"""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import build_ref, capi
from tests.cases import sample_indices
from tests.test_ref_kernels_gpu import _dcn_inputs

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refk_deform_conv_f16.npz")
FLOOR = 2.0 ** -10
NAMES = ("output", "grad_input", "grad_weight", "grad_bias", "grad_offset", "grad_mask")
CASES = [
    # B, C, H, W, Cout, k, s, p, d, group, dg, with_bias, big_offset
    (2, 128, 16, 16, 128, 3, 1, 1, 1, 1, 1, True, False),     # fused, full 8 x 16 tiles
    (2, 128, 13, 19, 128, 3, 2, 1, 1, 1, 1, False, True),     # fused, stride 2 with input-sized offsets, ragged tiles
    (1, 256, 9, 20, 128, 3, 1, 1, 1, 1, 1, True, False),      # fused, two 128-channel chunks per tap
    (2, 8, 9, 11, 8, 3, 1, 1, 1, 1, 1, True, False),          # outside the fused path: fp32 kernels on fp32 copies
]


def _inputs(case, cuda):
    B, C, H, W, Cout, k, s, p, d, group, dg, with_bias, big = case
    arrs = _dcn_inputs(21, B, C, H, W, Cout, k, s, p, d, group, dg, big)[:6]
    return [torch.from_numpy(a).to(cuda, torch.float16) for a in arrs]


def _run_reference(ref, case, t):
    B, C, H, W, Cout, k, s, p, d, group, dg, with_bias, big = case
    tx, tw, tb, toff, tm, tgo = t
    e = lambda: tx.new_empty(0)  # noqa: E731
    out = tx.new_empty(tgo.shape)
    ref.modulated_deform_conv_cuda_forward(tx, tw, tb, e(), toff, tm, out, e(), k, k, s, s, p, p, d, d, group, dg, with_bias)
    gi, gw, gb, goff, gm = [torch.zeros_like(a) for a in (tx, tw, tb, toff, tm)]
    ref.modulated_deform_conv_cuda_backward(tx, tw, tb, e(), toff, tm, e(), gi, gw, gb, goff, gm, tgo, k, k, s, s, p, p, d, d,
                                            group, dg, with_bias)
    torch.cuda.synchronize()
    return dict(zip(NAMES, (out, gi, gw, gb, goff, gm)))


def _run_ours(case, t):
    from megreader_b200 import dcn
    B, C, H, W, Cout, k, s, p, d, group, dg, with_bias, big = case
    tx, tw, tb, toff, tm, tgo = t
    out = tx.new_empty(tgo.shape)
    dcn.modulated_deform_conv_cuda_forward(tx, tw, tb, None, toff, tm, out, None, k, k, s, s, p, p, d, d, group, dg, with_bias)
    gi, gw, gb, goff, gm = [torch.zeros_like(a) for a in (tx, tw, tb, toff, tm)]
    dcn.modulated_deform_conv_cuda_backward(tx, tw, tb, None, toff, tm, None, gi, gw, gb, goff, gm, tgo, k, k, s, s, p, p, d, d,
                                            group, dg, with_bias)
    return dict(zip(NAMES, (out, gi, gw, gb, goff, gm)))


def _oracle(case, t):
    B, C, H, W, Cout, k, s, p, d, group, dg, with_bias, big = case
    x, w, b, off, m, go = [a.double().cpu().numpy() for a in t]
    geo = (s, p, d, group, dg)
    out = capi.dcn_forward(x, w, b if with_bias else None, off, m, *geo)
    gi, gw, gb, goff, gm = capi.dcn_backward(x, w, b if with_bias else None, off, m, go, *geo)
    return dict(zip(NAMES, (out, gi, gw, gb, goff, gm)))


def _flat(a):
    return (a.double().cpu().numpy() if torch.is_tensor(a) else np.asarray(a, np.float64)).reshape(-1)


def _rel(a, ref):
    return float(np.linalg.norm(a - ref) / max(np.linalg.norm(ref), 1e-300))


def _names(case):
    return [n for n in NAMES if n != "grad_bias" or case[11]]


@pytest.mark.parametrize("idx", range(len(CASES)))
def test_dcnv2_f16_vs_reference_kernels(cuda, idx):
    case = CASES[idx]
    t = _inputs(case, cuda)
    ours, orc = _run_ours(case, t), _oracle(case, t)
    for n in _names(case):
        assert ours[n].dtype == torch.float16 and torch.isfinite(ours[n]).all(), n
    sources = []
    with np.load(GOLD) as g:
        stored = {n: (g["%d.%s" % (idx, n)].astype(np.float64),
                      g["%d.%s__idx" % (idx, n)] if "%d.%s__idx" % (idx, n) in g.files else None) for n in _names(case)}
    sources.append(("stored sample", stored))
    mod = build_ref.load("ref_deform_conv")
    if mod is not None:
        live = _run_reference(mod, case, t)
        sources.append(("live", {n: (_flat(live[n]), None) for n in _names(case)}))
    for what, refk in sources:
        for n in _names(case):
            r, sel = refk[n]
            mine, o = _flat(ours[n]), _flat(orc[n])
            if sel is not None:
                mine, o = mine[sel], o[sel]
            e_ours, e_ref = _rel(mine, o), _rel(r, o)
            print("case %d %s %s: ours %.3g, reference %.3g (vs float64)" % (idx, what, n, e_ours, e_ref))
            assert e_ours <= max(e_ref, FLOOR), ("case %d %s: relative L2 error %.3g against float64 exceeds the reference "
                                                 "kernels' %.3g and the fp16 floor %.3g" % (idx, n, e_ours, e_ref, FLOOR))


def record(out_dir):
    """Run the reference's fp16 kernels on every case and store a sample of each array (needs a GPU and oracle/_ref)."""
    mod = build_ref.load("ref_deform_conv")
    assert mod is not None, "oracle/_ref/ref_deform_conv.so is not built (python -m oracle.build_ref)"
    cuda = torch.device("cuda:0")
    store = {}
    for idx, case in enumerate(CASES):
        live = _run_reference(mod, case, _inputs(case, cuda))
        for n in _names(case):
            a = live[n].cpu().numpy().reshape(-1)
            sel = sample_indices(a.astype(np.float32))
            store["%d.%s" % (idx, n)] = a.copy() if sel is None else a[sel]
            if sel is not None:
                store["%d.%s__idx" % (idx, n)] = sel.astype(np.int32)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, os.path.basename(GOLD))
    np.savez_compressed(path, **store)
    print(path, len(store), "arrays")


if __name__ == "__main__":
    record(sys.argv[1])
