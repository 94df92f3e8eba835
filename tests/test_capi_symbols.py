"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol include/*.h declares
(no compute calls — there is no GPU here)."""
import ctypes
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def so_path():
    from megreader_b200 import build
    return build.build()


def declared_symbols():
    names = []
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        text = open(h).read()
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        names += re.findall(r"\b(mr_[a-z0-9_]+)\s*\(", text)
    return sorted(set(names))


def test_header_declares_entry_points():
    syms = declared_symbols()
    assert "mr_ctc2d_forward_f32" in syms and "mr_ctc2d_backward_f32" in syms


def test_library_exports_every_declared_symbol(so_path):
    L = ctypes.CDLL(so_path)
    missing = [s for s in declared_symbols() if not hasattr(L, s)]
    assert not missing, missing


def test_ctypes_table_matches_header(so_path):
    from megreader_b200 import _lib
    assert sorted(_lib._SIGS) == declared_symbols()
    L = _lib.lib()
    assert L.mr_abi_version() >= 1
    assert L.mr_status_string(2) == b"blank must be in label range"


def test_argument_validation_without_gpu(so_path):
    """Pure host-side checks return before any CUDA call."""
    from megreader_b200 import _lib
    L = _lib.lib()
    # blank out of range -> MR_ERR_BLANK_RANGE (ctc2d_cuda.cu:40)
    rc = L.mr_ctc2d_forward_f32(1, 1, 1, 1, 4, 2, 1, 5, 3, 3, 1, 7, 0, 1, 1, None)
    assert rc == 2
    # 2S+1 > 1024 -> MR_ERR_TARGET_TOO_LONG (ctc2d_cuda_kernel.cu:220)
    rc = L.mr_ctc2d_forward_f32(1, 1, 1, 1, 4, 2, 1, 5, 600, 600, 1, 0, 0, 1, 1, None)
    assert rc == 3
    # empty batch is a no-op
    assert L.mr_ctc2d_forward_f32(None, None, None, None, 4, 2, 0, 5, 3, 3, 1, 0, 0, None, None, None) == 0
    # wgmma GEMM: every split-K CTA runs the epilogue, so bias with splits > 1 and ReLU with beta = 1 are refused
    # (aligned dummy pointers: the checks come before anything touches them)
    A, B, C, bias = 0x10000, 0x20000, 0x30000, 0x40000
    gemm = lambda transA, transB, bias, relu, beta, splits: L.mr_gemm_tcgen05(  # noqa: E731
        A, B, C, 256, 256, 1024, 1024, 1024, 256, transA, transB, 0, bias, relu, beta, splits, None)
    assert gemm(0, 1, bias, 0, 1.0, 2) == _lib.MR_ERR_UNSUPPORTED
    assert gemm(1, 0, bias, 0, 1.0, 4) == _lib.MR_ERR_UNSUPPORTED
    assert gemm(0, 1, None, 1, 1.0, 1) == _lib.MR_ERR_UNSUPPORTED
    assert gemm(0, 0, bias, 1, 1.0, 1) == _lib.MR_ERR_UNSUPPORTED
    assert gemm(1, 1, None, 0, 0.0, 1) == _lib.MR_ERR_UNSUPPORTED      # (transA, transB) = (1, 1)
    assert gemm(0, 1, None, 0, 0.5, 1) == _lib.MR_ERR_UNSUPPORTED


def test_dcn_fused_workspace_sizes(so_path):
    """The five fused-DCN workspace sizes against their closed forms: r() rounds a piece up to 256 bytes; the pieces are the
    NHWC input copy, the fp32 NHWC grad_input scratch, the re-tiled grad_output and the packed weights (bf16 hi and lo for
    fp32, one copy for half precision), and for half precision the fp32 bias copy and grad_weight scratch."""
    import itertools
    from megreader_b200 import _lib
    L = _lib.lib()
    r = lambda n: -(-n // 256) * 256  # noqa: E731
    shapes = itertools.product((1, 3, 8), (64, 127, 256, 512), ((7, 9), (33, 65), (64, 64)), (128, 384), (1, 3, 5),
                               ((1, 1), (7, 15), (9, 17), (32, 64), (33, 65)))
    for B, C, (H, W), Cout, k, (Ho, Wo) in shapes:
        K, tiles = k * k, -(-Wo // 16) * -(-Ho // 8)
        x4, g, w = r(4 * B * H * W * C), r(256 * B * tiles * Cout), r(2 * Cout * C * K)
        shape = (B, C, H, W, Cout, k, k, Ho, Wo)
        assert L.mr_dcn_fused_workspace_bytes(B, C, H, W, Cout, k, k) == x4 + 2 * w, shape
        assert L.mr_dcn_fused_wgrad_workspace_bytes(B, C, H, W, Cout, Ho, Wo) == x4 + 2 * g, shape
        assert L.mr_dcn_fused_backward_workspace_bytes(B, C, H, W, Cout, Ho, Wo, k, k) == 2 * x4 + 2 * g + 2 * w, shape
        assert L.mr_dcn_fused_workspace_bytes_h(B, C, H, W, Cout, k, k) == r(2 * B * H * W * C) + w + r(4 * Cout), shape
        assert (L.mr_dcn_fused_backward_workspace_bytes_h(B, C, H, W, Cout, Ho, Wo, k, k)
                == r(2 * B * H * W * C) + x4 + g + w + r(4 * Cout * C * K)), shape


def test_product_never_imports_oracle():
    for path in glob.glob(os.path.join(ROOT, "megreader_b200", "**", "*.py"), recursive=True):
        src = open(path).read()
        assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), path
