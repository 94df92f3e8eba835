"""megreader_b200 — H100-native (sm_90a) rebuild of MegReader's recognition hot path.

Host code is Python/PyTorch (device memory, streams, torch.distributed); all arithmetic on the
path runs in hand-written CUDA reached through the C-ABI in include/megreader_b200.h
(libmegreader_b200.so, bound with ctypes in megreader_b200/_lib.py).  No CPU fallback.

    import megreader_b200
    megreader_b200.install_reference_api()   # exposes `ops`, `decoders`, `backbones`, `assets.ops.dcn`
                                             # under the reference's own import paths
"""
from . import _lib  # noqa: F401
from ._lib import MegReaderB200Error, launch_count, reset_launch_count  # noqa: F401

__version__ = "0.1.0"


def install_reference_api():
    from .refapi import install
    return install()
