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


def test_product_never_imports_oracle():
    for path in glob.glob(os.path.join(ROOT, "megreader_b200", "**", "*.py"), recursive=True):
        src = open(path).read()
        assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), path
