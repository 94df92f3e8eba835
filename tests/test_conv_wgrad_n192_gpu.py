"""The weight gradient on 128 x 192 tiles (csrc/conv_pingpong.cu, conv_wgrad_n192_kernel), which the CRNN engine runs where
kh*kw*C is a multiple of 192 but not of 256 (L1 and L2).  Against float64 conv2d_weight on the same bf16 operands within
tests.wgmma_variants.bound at small batches: Cout = 192 (half a 128-row tile), a column tile that runs past K, both K-block
heights (RB = 64 and 80 output pixels), ragged image remainders; at L1 and L2 at N = 512 against conv_wgrad_tcgen05_kernel
within twice the bound.  A bf16 CRNN step must run it at L1 and L2 only, and a CPU test checks that every compiled instantiation is the
expected kernel of one of these cases."""
import re
import shutil

import pytest
import torch

from tests import wgmma_variants as wv

# (name, input H, W, C, Cout, k, padding) of the CRNN layers whose K = 9 * C is 576 and 1152
LAYERS = [("L1", 16, 128, 64, 128, 3, 1), ("L2", 8, 64, 128, 256, 3, 1)]
# (k, padding, C, Cout, Ho, Wo, N): K = 576 / 1152 / 256 (the second 192-column tile holds one real atom), Cout = 192,
# Wo = 64 and 128 (RB = 64), 65 and 80 (RB = 80, several K-block segments), batches that leave partial image blocks
EDGE = [(3, 1, 64, 192, 4, 64, 3), (3, 1, 64, 128, 2, 128, 37), (3, 1, 128, 192, 1, 65, 81), (3, 1, 128, 256, 2, 80, 5),
        (2, 0, 64, 192, 2, 66, 37), (2, 0, 64, 128, 1, 64, 1), (3, 1, 64, 64, 3, 72, 7), (3, 1, 128, 192, 4, 128, 3)]


def expected_kernel(Wo):
    """RB = 80 output pixels per K block iff 64 < Wo <= 80, as for conv_wgrad_pp_kernel."""
    return "conv_wgrad_n192_kernel<%d>" % (80 if 64 < Wo <= 80 else 64)


def _ref(x, dz, Cout, C, k, p):
    """float64 conv2d_weight as [Cout, k*k*C], columns (tap, channel) like the kernel's"""
    w = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (Cout, C, k, k), dz.double().permute(0, 3, 1, 2),
                                    padding=p)
    return w.permute(0, 2, 3, 1).reshape(Cout, -1)


@pytest.mark.gpu
@pytest.mark.parametrize("k,p,C,Cout,Ho,Wo,n", EDGE,
                         ids=["k%d-C%d-Cout%d-Ho%d-Wo%d-N%d" % ((c[0],) + c[2:]) for c in EDGE])
def test_n192_wgrad_within_bound(cuda, k, p, C, Cout, Ho, Wo, n):
    from megreader_b200 import nnops
    H, W = Ho + k - 1 - 2 * p, Wo + k - 1 - 2 * p
    g = torch.Generator(device=cuda).manual_seed(1000 * Wo + 10 * n + k + C)
    x = torch.randn((n, H, W, C), generator=g, device=cuda).bfloat16()
    dz = torch.randn((n, Ho, Wo, Cout), generator=g, device=cuda).bfloat16()
    got = nnops.conv_wgrad_n192(dz, x, k, k, p, p)
    assert got is not None, "conv_wgrad_n192 refused the geometry"
    wv.assert_within(got, _ref(x, dz, Cout, C, k, p), wv.bound(_ref(x.abs(), dz.abs(), Cout, C, k, p)),
                     "n192 wgrad k=%d C=%d Cout=%d Ho=%d Wo=%d N=%d" % (k, C, Cout, Ho, Wo, n))


def _spy(monkeypatch):
    """Records the geometries the engine sends to nnops.conv_wgrad_n192 (no profiler: many profiler sessions in one
    process were seen to lose kernel records, see tests/wgmma_variants.run_variant)."""
    from megreader_b200 import nnops
    seen, real = [], nnops.conv_wgrad_n192

    def spy(dz, x, kh, kw, ph, pw, **kw_):
        seen.append((x.size(3), dz.size(3), kh, kw))
        return real(dz, x, kh, kw, ph, pw, **kw_)
    monkeypatch.setattr(nnops, "conv_wgrad_n192", spy)
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("lay", LAYERS, ids=[x[0] for x in LAYERS])
def test_engine_wgrad_at_l1_l2_against_one_tile_kernel(cuda, lay, monkeypatch):
    from megreader_b200 import crnn_engine, nnops
    name, H, W, C, Cout, k, p = lay
    n = 512
    Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
    g = torch.Generator(device=cuda).manual_seed(17 * k + C)
    x = torch.randn((n, H, W, C), generator=g, device=cuda).bfloat16()
    dz = torch.randn((n, Ho, Wo, Cout), generator=g, device=cuda).bfloat16()
    want = nnops.conv_wgrad_tc(dz, x, k, k, p, p)
    bnd = 2 * wv.bound(nnops.conv_wgrad_tc(dz.abs(), x.abs(), k, k, p, p).double())
    seen = _spy(monkeypatch)
    got = crnn_engine._conv_wgrad(dz, x, k, k, p, p)
    assert seen == [(C, Cout, k, k)]
    wv.assert_within(got, want, bnd, "engine wgrad %s N=%d" % (name, n))


@pytest.mark.gpu
def test_bf16_crnn_step_runs_the_192_column_kernel(cuda, monkeypatch):
    """L1 and L2 (K = 576, 1152) go to the 192-column entry, and no other layer does."""
    from tests.test_conv_pingpong_gpu import _crnn
    step = _crnn(cuda)
    seen = _spy(monkeypatch)
    step()
    torch.cuda.synchronize()
    assert sorted(seen) == [(64, 128, 3, 3), (128, 256, 3, 3)], seen


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None,
                    reason="needs cuobjdump and cu++filt from the CUDA toolkit")
def test_every_n192_instantiation_has_a_gpu_case():
    from megreader_b200 import build
    from tests.test_kernel_inventory import compiled_kernels
    found = {n for n in map(wv.normalise, compiled_kernels(build.build())) if re.fullmatch(r"conv_wgrad_n192_kernel<\d+>", n)}
    covered = {expected_kernel(c[5]) for c in EDGE}
    assert found, "no conv_wgrad_n192_kernel instantiation compiled"
    assert found == covered, "compiled: %s; expected by a GPU case: %s" % (sorted(found), sorted(covered))
