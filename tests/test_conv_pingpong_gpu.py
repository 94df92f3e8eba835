"""The persistent convolution kernels (csrc/conv_pingpong.cu) against the one-tile-per-CTA kernels they replace in the CRNN
engine: forward and input gradient at the six CRNN layer geometries must give the same bits as conv_fprop_tcgen05_kernel
(same K order, same wgmma shape, same rounding); the weight gradient (fp32 atomics, so no fixed summation order) must lie
within tests.wgmma_variants.bound of float64 conv2d_weight at small batches and of conv_wgrad_tcgen05_kernel at N = 512.
A CPU test checks that every compiled instantiation is the expected kernel of one of these cases; which instantiations a
bf16 training step launches is checked once, under torch.profiler (many profiler sessions in one process were seen to lose
kernel records, see tests/wgmma_variants.run_variant)."""
import re
import shutil

import pytest
import torch

from tests import wgmma_variants as wv

# (name, input H, W, C, Cout, k, padding) of the implicit convolutions of backbones/crnn.py at 32 x 256 lines
LAYERS = [("L1", 16, 128, 64, 128, 3, 1), ("L2", 8, 64, 128, 256, 3, 1), ("L3", 8, 64, 256, 256, 3, 1),
          ("L4", 4, 65, 256, 512, 3, 1), ("L5", 4, 65, 512, 512, 3, 1), ("L6", 2, 66, 512, 512, 2, 0)]
# 512: the bench batch; 3: partial tiles in every segment (and the 1-wide Wo = 65 segment of 32 images holds 3); 37: tile
# counts that are not multiples of the 132-CTA grid, so the CTAs own different numbers of tiles (odd and even)
BATCHES = [512, 3, 37]
CASES = [(lay, kind, n) for lay in LAYERS for kind in ("fprop", "dgrad") for n in BATCHES]


def expected_kernel(lay, kind):
    """BN = 128 when the convolution's output has more than 64 channels (the input gradient's output has C channels)."""
    _, H, W, C, Cout, k, p = lay
    cout = Cout if kind == "fprop" else C
    return "conv_fprop_pp_kernel<%d>" % (128 if cout > 64 else 64)


def expected_wgrad_kernel(lay):
    """RB = 80 output pixels per K block iff 64 < Wo <= 80."""
    _, H, W, C, Cout, k, p = lay
    Wo = W + 2 * p - k + 1
    return "conv_wgrad_pp_kernel<%d>" % (80 if 64 < Wo <= 80 else 64)


WGRAD_CASES = [(lay, n) for lay in LAYERS for n in (3, 37, 512)]


def _operands(lay, kind, n, dev):
    _, H, W, C, Cout, k, p = lay
    g = torch.Generator(device=dev).manual_seed(n * 7 + k)
    Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
    if kind == "fprop":
        x = torch.randn((n, H, W, C), generator=g, device=dev).bfloat16()
        Wm = (torch.randn((Cout, k * k * C), generator=g, device=dev) / (k * k * C) ** 0.5).bfloat16()
        return x, Wm, k, p
    dz = torch.randn((n, Ho, Wo, Cout), generator=g, device=dev).bfloat16()
    Wd = (torch.randn((C, k * k * Cout), generator=g, device=dev) / (k * k * Cout) ** 0.5).bfloat16()
    return dz, Wd, k, k - 1 - p


@pytest.mark.gpu
@pytest.mark.parametrize("lay,kind,n", CASES, ids=["%s-%s-N%d" % (c[0][0], c[1], c[2]) for c in CASES])
def test_pingpong_bit_identical_to_one_tile_kernel(cuda, lay, kind, n):
    from megreader_b200 import nnops
    x, Wm, k, pad = _operands(lay, kind, n, cuda)
    want, Ho, Wo = nnops.conv_fprop_tc(x, Wm, k, k, pad, pad)
    r = nnops.conv_fprop_pp(x, Wm, k, k, pad, pad)
    assert r is not None, "conv_fprop_pp refused a CRNN geometry"
    got, Hp, Wp = r
    assert (Hp, Wp) == (Ho, Wo)
    diff = (got.float() - want.float()).abs()
    assert torch.equal(got, want), "%d of %d elements differ, worst %g" % (int((diff > 0).sum()), diff.numel(),
                                                                          float(diff.max()))


@pytest.mark.gpu
@pytest.mark.parametrize("lay,n", WGRAD_CASES, ids=["%s-N%d" % (c[0][0], c[1]) for c in WGRAD_CASES])
def test_wgrad_within_bound(cuda, lay, n):
    """Small batches: against float64 conv2d_weight on the same bf16 operands.  N = 512: against the one-tile-per-CTA
    kernel; each of the two errs by at most the bound, so they differ by at most twice that."""
    from megreader_b200 import nnops
    _, H, W, C, Cout, k, p = lay
    g = torch.Generator(device=cuda).manual_seed(n * 11 + k)
    Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
    x = torch.randn((n, H, W, C), generator=g, device=cuda).bfloat16()
    dz = torch.randn((n, Ho, Wo, Cout), generator=g, device=cuda).bfloat16()
    got = nnops.conv_wgrad_pp(dz, x, k, k, p, p)
    assert got is not None, "conv_wgrad_pp refused a CRNN geometry"
    if n < 512:
        def ref(a, b):      # [Cout, k*k*C], columns (tap, channel) like the kernel's
            w = torch.nn.grad.conv2d_weight(a.double().permute(0, 3, 1, 2), (Cout, C, k, k), b.double().permute(0, 3, 1, 2),
                                            padding=p)
            return w.permute(0, 2, 3, 1).reshape(Cout, -1)
        want, bnd = ref(x, dz), wv.bound(ref(x.abs(), dz.abs()))
    else:
        want = nnops.conv_wgrad_tc(dz, x, k, k, p, p)
        bnd = 2 * wv.bound(nnops.conv_wgrad_tc(dz.abs(), x.abs(), k, k, p, p).double())
    wv.assert_within(got, want, bnd, "wgrad %s N=%d" % (lay[0], n))


@pytest.mark.gpu
def test_unsupported_geometry_is_refused(cuda):
    """C % 64 != 0 has no TMA box of 64 channels: the entry refuses it and conv_fprop_pp hands back None."""
    from megreader_b200 import nnops
    x = torch.randn((2, 8, 8, 32), device=cuda).bfloat16()
    Wm = torch.randn((64, 9 * 32), device=cuda).bfloat16()
    assert nnops.conv_fprop_pp(x, Wm, 3, 3, 1, 1) is None
    assert nnops.conv_wgrad_pp(torch.randn((2, 8, 8, 64), device=cuda).bfloat16(), x, 3, 3, 1, 1) is None


def _crnn(cuda):
    import megreader_b200
    from tests.weights import crnn_batch, fill_state_dict
    megreader_b200.install_reference_api()
    import backbones
    import decoders
    bb = fill_state_dict(backbones.crnn_backbone(), "bb.").to(cuda).train()
    dec = fill_state_dict(decoders.CRNNDecoder(in_channels=512, inner_channels=256), "dec.").to(cuda).train()
    x, labels, lengths = [torch.from_numpy(a).to(cuda) for a in crnn_batch(0, 8, 256, 16, 65)]
    state = {k: v.clone() for k, v in bb.state_dict().items()}

    def step():
        """one bf16 training step from the same BatchNorm state; -> the backbone's weight gradients"""
        from megreader_b200 import crnn_engine
        bb.load_state_dict(state)
        for q in bb.parameters():
            q.grad = None
        crnn_engine.set_compute_dtype(torch.bfloat16)
        try:
            loss, _ = dec(bb(x), targets=labels, lengths=lengths, train=True)
            loss.mean().backward()
        finally:
            crnn_engine.set_compute_dtype(torch.float32)
        return {n: q.grad.clone() for n, q in bb.named_parameters() if n.endswith("weight") and q.dim() == 4}
    return step


@pytest.mark.gpu
def test_bf16_crnn_step_runs_the_persistent_kernels(cuda):
    step = _crnn(cuda)
    step()
    _, names = wv.launched_kernels(step)
    assert {"conv_fprop_pp_kernel<64>", "conv_fprop_pp_kernel<128>", "conv_wgrad_pp_kernel<64>",
            "conv_wgrad_pp_kernel<80>"} <= names, sorted(names)
    assert not [nm for nm in names if nm.startswith(("conv_fprop_tcgen05_kernel", "conv_wgrad_tcgen05_kernel"))], sorted(names)


@pytest.mark.gpu
def test_wgrad_side_stream_gives_the_same_gradients(cuda, monkeypatch):
    """MEGREADER_B200_WGRAD_STREAM=1 (off by default): the weight gradients run on a side stream and are joined before
    they are handed back; they must equal the in-order ones up to the order of the fp32 atomics."""
    from megreader_b200 import crnn_engine
    step = _crnn(cuda)
    monkeypatch.setattr(crnn_engine, "WGRAD_SIDE_STREAM", False)
    want = step()
    monkeypatch.setattr(crnn_engine, "WGRAD_SIDE_STREAM", True)
    got = step()
    torch.cuda.synchronize()
    assert sorted(got) == sorted(want) and len(want) == 7
    for n in want:
        torch.testing.assert_close(got[n], want[n], rtol=1e-4, atol=1e-5 * float(want[n].abs().max()), msg=n)


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None,
                    reason="needs cuobjdump and cu++filt from the CUDA toolkit")
def test_every_pingpong_instantiation_has_a_gpu_case():
    from megreader_b200 import build
    from tests.test_kernel_inventory import compiled_kernels
    found = {n for n in map(wv.normalise, compiled_kernels(build.build())) if re.fullmatch(r"conv_\w+_pp_kernel<[\d,]+>", n)}
    covered = {expected_kernel(lay, kind) for lay, kind, _ in CASES} | {expected_wgrad_kernel(lay) for lay, _ in WGRAD_CASES}
    assert found, "no conv_*_pp_kernel instantiation compiled"
    assert found == covered, "compiled: %s; expected by a GPU case: %s" % (sorted(found), sorted(covered))
