"""Baseline JPEG decoding on the device (csrc/jpeg.cu), equal to cv2.imdecode(buf, cv2.IMREAD_COLOR) bit for bit.

    pack_bytes(blobs)                                   -> (data uint8, offsets int64 [N + 1]) on the device, one copy
    decode_packed(data, offsets, max_h, max_w, cap)     -> dict(buffer, image_offsets, shapes, status) in db_batch's packed
                                                           layout; never synchronises with the host, so it can be captured
                                                           in a CUDA graph and replayed with new bytes in the same tensors
    decode(blobs)                                       -> (list of HWC uint8 CUDA views, status int32 [N] on the host)

Baseline and extended-sequential Huffman files with 8-bit samples in one interleaved scan: grey or three components
(YCbCr, or RGB by libjpeg's colour-space rule), every integral sampling layout, restart intervals, EXIF orientation.  Other
files get a STATUS bit, shape (0, 0) and no pixels; the other images of the batch are unaffected.  CUDA only; no CPU
fallback."""
import torch

from . import _lib

STATUS = dict(bad_header=1, unsupported_process=2, unsupported_components=4, too_large=8, corrupt=16, bad_offsets=32)
MAX_SIDE = 16384


def _stream():
    return torch.cuda.current_stream().cuda_stream


def pack_bytes(blobs, device=None):
    """Host byte strings -> (data uint8 [total], offsets int64 [N + 1]) on the device: one pinned buffer, one copy each."""
    if not blobs:
        raise ValueError("jpeg.pack_bytes: need at least one image")
    device = torch.device(device if device is not None else "cuda")
    sizes = [len(b) for b in blobs]
    host = torch.empty(max(sum(sizes), 1), dtype=torch.uint8, pin_memory=True)
    offs = torch.zeros(len(blobs) + 1, dtype=torch.int64, pin_memory=True)
    pos = 0
    for i, b in enumerate(blobs):
        if sizes[i]:
            host[pos:pos + sizes[i]] = torch.frombuffer(bytearray(b), dtype=torch.uint8)
        pos += sizes[i]
        offs[i + 1] = pos
    return host.to(device, non_blocking=True), offs.to(device, non_blocking=True)


def workspace_bytes(n, byte_capacity, pixel_capacity):
    return int(_lib.lib().mr_jpeg_workspace_bytes(n, byte_capacity, pixel_capacity))


def decode_packed(data, offsets, max_h, max_w, pixel_capacity, out=None):
    """Decode the N images of data (uint8, device) at offsets (int64 [N + 1], device).  Returns dict(buffer uint8
    [3 * pixel_capacity] HWC BGR, image_offsets int64 [N] in elements, shapes int32 [N, 2] as (h, w), status int32 [N],
    workspace).  Images with a side above max_h / max_w, or past pixel_capacity, are flagged (STATUS too_large).  `out`, a
    dict returned by an earlier call of the same sizes, is filled again in place (for graph replay).  No host
    synchronisation."""
    for name, t in (("data", data), ("offsets", offsets)):
        if not (torch.is_tensor(t) and t.is_cuda):
            raise NotImplementedError("megreader_b200: jpeg runs on CUDA only (no CPU fallback); %s is not a CUDA tensor" % name)
    if data.dtype != torch.uint8 or data.dim() != 1 or offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.numel() < 2:
        raise RuntimeError("jpeg.decode_packed: data must be flat uint8 and offsets int64 [N + 1]")
    N = offsets.numel() - 1
    cap = int(pixel_capacity)
    dev = data.device
    nbytes = data.numel()
    if out is None:
        wsb = workspace_bytes(N, nbytes, cap)
        if wsb <= 0:
            raise RuntimeError("jpeg.decode_packed: bad sizes (N = %d, %d bytes, pixel capacity %d)" % (N, nbytes, cap))
        out = dict(buffer=torch.empty(max(3 * cap, 1), dtype=torch.uint8, device=dev),
                   image_offsets=torch.empty(N, dtype=torch.int64, device=dev),
                   shapes=torch.empty((N, 2), dtype=torch.int32, device=dev),
                   status=torch.empty(N, dtype=torch.int32, device=dev),
                   workspace=torch.empty(wsb, dtype=torch.uint8, device=dev))
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().mr_jpeg_decode(data.data_ptr(), nbytes, offsets.data_ptr(), N, int(max_h), int(max_w), cap,
                                             out["workspace"].data_ptr(), out["workspace"].numel(), out["buffer"].data_ptr(),
                                             out["image_offsets"].data_ptr(), out["shapes"].data_ptr(), out["status"].data_ptr(),
                                             _stream()),
                   "jpeg_decode")
    return out


def decode(blobs, max_h=MAX_SIDE, max_w=MAX_SIDE, pixel_capacity=None, device=None):
    """The one-call form of cv2.imdecode(buf, cv2.IMREAD_COLOR) for a list of byte strings: (list of HWC uint8 CUDA views,
    None for a flagged image; status int32 [N] numpy).  pixel_capacity defaults to a bound from the headers (one host read)."""
    data, offsets = pack_bytes(blobs, device)
    if pixel_capacity is None:
        pixel_capacity = sum(_header_pixels(b) for b in blobs)
    res = decode_packed(data, offsets, max_h, max_w, max(int(pixel_capacity), 1))
    shapes = res["shapes"].cpu().tolist()
    offs = res["image_offsets"].cpu().tolist()
    status = res["status"].cpu().numpy()
    views = []
    for (h, w), o, s in zip(shapes, offs, status):
        views.append(res["buffer"][o:o + h * w * 3].view(h, w, 3) if s == 0 else None)
    return views, status


def _header_pixels(blob):
    """h * w from the first SOF marker of a byte string (0 when there is none); only sizes the output buffer"""
    b = bytes(blob)
    i = 2
    while i + 9 < len(b):
        if b[i] != 0xFF:
            i += 1
            continue
        m = b[i + 1]
        if m == 0xFF:
            i += 1
            continue
        if 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            return int.from_bytes(b[i + 5:i + 7], "big") * int.from_bytes(b[i + 7:i + 9], "big")
        if m == 0xDA or m == 0xD9:
            return 0
        i += 2 + int.from_bytes(b[i + 2:i + 4], "big")
    return 0
