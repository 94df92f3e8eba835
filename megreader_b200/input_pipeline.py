"""Recognition input step on the GPU (SURVEY.md §8 row N3): what `ResizeImage` (modes "resize" / "pad") + `NormalizeImage`
(data/processes/resize_image.py:29-57, normalize_image.py:10-17) and `MakeRecognitionLabel`
(make_recognition_label.py:13-32) do per sample on the host, for a whole ragged batch in one launch each
(csrc/input_pipeline.cu through the C-ABI).  CUDA only; no CPU fallback."""
import ctypes

import numpy as np
import torch

from . import _lib
from .charset import default_charset

RGB_MEAN = (122.67891434, 116.66876762, 104.00698793)              # normalize_image.py:8 (applied in stored channel order)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def resized_width(mode, image_size, src_h, src_w):
    """resize_image.py:41-48 (destination width of one image; the canvas is image_size)"""
    height, width = image_size
    if mode == "pad":
        width = min(width, max(int(height / src_h * src_w / 32 + 0.5) * 32, 32))
    elif mode != "resize":
        raise ValueError("batched input step supports modes 'resize' and 'pad' (fixed-size outputs), got %r" % (mode,))
    return width


def resize_normalize(images, image_size, mode="resize", device=None, mean=RGB_MEAN):
    """images: list of HWC 3-channel numpy arrays (uint8 as decoded, or float32), any sizes -> float32 CUDA tensor
    [N, 3, H, W] = NormalizeImage(ResizeImage(image_size, mode)(image.astype('float32')))."""
    device = torch.device(device if device is not None else "cuda")
    if device.type != "cuda":
        raise NotImplementedError("megreader_b200: the input step runs on CUDA only (no CPU fallback)")
    n = len(images)
    dst_h, dst_w = int(image_size[0]), int(image_size[1])
    out = torch.empty((n, 3, dst_h, dst_w), dtype=torch.float32, device=device)
    if n == 0:
        return out
    u8 = all(im.dtype == np.uint8 for im in images)
    dt = np.uint8 if u8 else np.float32
    flat, offsets, hs, ws, valid = [], [0], [], [], []
    for im in images:
        if im.ndim != 3 or im.shape[2] != 3:
            raise RuntimeError("expected HWC images with 3 channels")
        a = np.ascontiguousarray(im, dtype=dt).reshape(-1)
        flat.append(a)
        offsets.append(offsets[-1] + a.size)
        hs.append(im.shape[0])
        ws.append(im.shape[1])
        valid.append(resized_width(mode, (dst_h, dst_w), im.shape[0], im.shape[1]))
    src = torch.from_numpy(np.concatenate(flat)).pin_memory().to(device, non_blocking=True)
    meta = torch.tensor(offsets[:-1], dtype=torch.int64).pin_memory().to(device, non_blocking=True)
    dims = torch.tensor([hs, ws, valid], dtype=torch.int32).pin_memory().to(device, non_blocking=True)
    mean3 = (ctypes.c_double * 3)(*mean)
    with torch.cuda.device(device):
        _lib.check(_lib.lib().mr_resize_normalize_f32(src.data_ptr(), int(u8), meta.data_ptr(), dims[0].data_ptr(),
                                                      dims[1].data_ptr(), dims[2].data_ptr(), n, dst_h, dst_w,
                                                      ctypes.cast(mean3, ctypes.c_void_p), out.data_ptr(), _stream()),
                   "resize_normalize")
    return out


def resize_normalize_packed(buffer, image_offsets, shapes, image_size, mode="resize", mean=RGB_MEAN):
    """resize_normalize of images already on the device in db_batch's packed layout (HWC uint8, as jpeg.decode_packed
    returns them): float32 [N, 3, H, W].  resized_width is computed on the device in float64 with the same expression, so
    there is no host read.  Rows of images with shape (0, 0) are zero."""
    for name, t in (("buffer", buffer), ("image_offsets", image_offsets), ("shapes", shapes)):
        if not (torch.is_tensor(t) and t.is_cuda):
            raise NotImplementedError("megreader_b200: the input step runs on CUDA only (no CPU fallback); %s is not a CUDA tensor" % name)
    if buffer.dtype != torch.uint8 or image_offsets.dtype != torch.int64 or shapes.dtype != torch.int32 or shapes.dim() != 2:
        raise RuntimeError("resize_normalize_packed: expected uint8 buffer, int64 image_offsets and int32 shapes [N, 2]")
    n = shapes.size(0)
    dst_h, dst_w = int(image_size[0]), int(image_size[1])
    out = torch.empty((n, 3, dst_h, dst_w), dtype=torch.float32, device=buffer.device)
    if n == 0:
        return out
    ok = shapes[:, 0] > 0
    hs = torch.where(ok, shapes[:, 0], 1).contiguous()
    ws = torch.where(ok, shapes[:, 1], 1).contiguous()
    offs = torch.where(ok, image_offsets, 0).contiguous()
    if mode == "pad":
        v = torch.trunc(dst_h / hs.double() * ws.double() / 32 + 0.5) * 32
        valid = torch.clamp(v, min=32, max=dst_w).to(torch.int32)
    elif mode == "resize":
        valid = torch.full_like(hs, dst_w)
    else:
        raise ValueError("batched input step supports modes 'resize' and 'pad' (fixed-size outputs), got %r" % (mode,))
    mean3 = (ctypes.c_double * 3)(*mean)
    with torch.cuda.device(buffer.device):
        _lib.check(_lib.lib().mr_resize_normalize_f32(buffer.data_ptr(), 1, offs.data_ptr(), hs.data_ptr(), ws.data_ptr(),
                                                      valid.data_ptr(), n, dst_h, dst_w, ctypes.cast(mean3, ctypes.c_void_p),
                                                      out.data_ptr(), _stream()),
                   "resize_normalize_packed")
    return out.mul_(ok.view(n, 1, 1, 1))


def charset_lut(charset=None):
    """256-entry byte -> class-index table of a charset (`Charset.index`, concern/charsets.py: unknown for anything else)."""
    charset = charset if charset is not None else default_charset()
    chars = getattr(charset, "_charset", None)          # the reference's Charset keeps its alphabet in `_charset` (concern/charsets.py)
    if chars is not None and any(ord(ch) > 255 for ch in chars if isinstance(ch, str) and len(ch) == 1):
        # e.g. the reference's ChineseCharset: a byte table would silently map every such character to `unknown`
        raise NotImplementedError("megreader_b200.input_pipeline.pack_labels: the charset has characters outside Latin-1; "
                                  "the GPU label packer works on a 256-entry byte table")
    return np.array([charset.index(chr(b)) for b in range(256)], dtype=np.int32)


def pack_labels(texts, charset=None, max_size=32, device=None):
    """list of ground-truth strings -> (labels int32 [N, max_size] blank-padded, lengths int32 [N]) on the GPU."""
    device = torch.device(device if device is not None else "cuda")
    if device.type != "cuda":
        raise NotImplementedError("megreader_b200: the input step runs on CUDA only (no CPU fallback)")
    n = len(texts)
    labels = torch.empty((n, max_size), dtype=torch.int32, device=device)
    lengths = torch.empty((n,), dtype=torch.int32, device=device)
    if n == 0:
        return labels, lengths
    raw = [t.encode("latin-1", "replace") for t in texts]
    offsets = np.zeros(n + 1, np.int64)
    offsets[1:] = np.cumsum([len(r) for r in raw])
    blob = np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8).copy()
    d_text = torch.from_numpy(blob).to(device)
    d_off = torch.from_numpy(offsets).to(device)
    d_lut = torch.from_numpy(charset_lut(charset)).to(device)
    with torch.cuda.device(device):
        _lib.check(_lib.lib().mr_pack_labels(d_text.data_ptr(), d_off.data_ptr(), n, d_lut.data_ptr(), max_size,
                                             labels.data_ptr(), lengths.data_ptr(), _stream()), "pack_labels")
    return labels, lengths
