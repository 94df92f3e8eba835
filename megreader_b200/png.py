"""PNG decoding on the device (csrc/png.cu), equal to cv2.imdecode(buf, cv2.IMREAD_COLOR) bit for bit.

    decode_packed(data, offsets, max_h, max_w, cap)     -> dict(buffer, image_offsets, shapes, status) in db_batch's packed
                                                           layout; never synchronises with the host (graph-capturable)
    decode(blobs)                                       -> (list of HWC uint8 CUDA views, status int32 [N] on the host)

The bytes are packed with jpeg.pack_bytes.  Every colour type and bit depth, Adam7, the eXIf orientation; 16-bit samples
reduced to their high byte, alpha and tRNS dropped, as cv2 does.  Other or broken files get a jpeg.STATUS bit, shape (0, 0)
and no pixels; the other images of the batch are unaffected.  CUDA only; no CPU fallback."""
import torch

from . import _lib
from .jpeg import MAX_SIDE, STATUS, pack_bytes  # noqa: F401  (the same status bits and packing as JPEG)


def workspace_bytes(n, byte_capacity, pixel_capacity):
    return int(_lib.lib().mr_png_workspace_bytes(n, byte_capacity, pixel_capacity))


def decode_packed(data, offsets, max_h, max_w, pixel_capacity, out=None):
    """as jpeg.decode_packed, for PNG files"""
    return _decode_packed_with("png", data, offsets, max_h, max_w, pixel_capacity, out)


def decode(blobs, max_h=MAX_SIDE, max_w=MAX_SIDE, pixel_capacity=None, device=None):
    """the one-call form of cv2.imdecode(buf, cv2.IMREAD_COLOR) for a list of PNG byte strings: (list of HWC uint8 CUDA
    views, None for a flagged image; status int32 [N] numpy).  pixel_capacity defaults to the sum over the IHDRs."""
    data, offsets = pack_bytes(blobs, device)
    if pixel_capacity is None:
        pixel_capacity = sum(header_pixels(b) for b in blobs)
    return _views(decode_packed(data, offsets, max_h, max_w, max(int(pixel_capacity), 1)))


def header_pixels(blob):
    """width * height from the IHDR of a byte string (0 when it is not a PNG); only sizes the output buffer"""
    b = bytes(blob[:24])
    if len(b) < 24 or b[:8] != b"\x89PNG\r\n\x1a\n" or b[12:16] != b"IHDR":
        return 0
    return int.from_bytes(b[16:20], "big") * int.from_bytes(b[20:24], "big")


def _decode_packed_with(kind, data, offsets, max_h, max_w, pixel_capacity, out=None):
    """mr_<kind>_decode (kind png or image) with jpeg.decode_packed's arguments, checks and result dict"""
    for name, t in (("data", data), ("offsets", offsets)):
        if not (torch.is_tensor(t) and t.is_cuda):
            raise NotImplementedError("megreader_b200: %s decode runs on CUDA only (no CPU fallback); %s is not a CUDA tensor"
                                      % (kind, name))
    if data.dtype != torch.uint8 or data.dim() != 1 or offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.numel() < 2:
        raise RuntimeError("%s.decode_packed: data must be flat uint8 and offsets int64 [N + 1]" % kind)
    L = _lib.lib()
    N = offsets.numel() - 1
    cap = int(pixel_capacity)
    dev = data.device
    nbytes = data.numel()
    if out is None:
        wsb = int(getattr(L, "mr_%s_workspace_bytes" % kind)(N, nbytes, cap))
        if wsb <= 0:
            raise RuntimeError("%s.decode_packed: bad sizes (N = %d, %d bytes, pixel capacity %d)" % (kind, N, nbytes, cap))
        out = dict(buffer=torch.empty(max(3 * cap, 1), dtype=torch.uint8, device=dev),
                   image_offsets=torch.empty(N, dtype=torch.int64, device=dev),
                   shapes=torch.empty((N, 2), dtype=torch.int32, device=dev),
                   status=torch.empty(N, dtype=torch.int32, device=dev),
                   workspace=torch.empty(wsb, dtype=torch.uint8, device=dev))
    with torch.cuda.device(dev):
        _lib.check(getattr(L, "mr_%s_decode" % kind)(
            data.data_ptr(), nbytes, offsets.data_ptr(), N, int(max_h), int(max_w), cap, out["workspace"].data_ptr(),
            out["workspace"].numel(), out["buffer"].data_ptr(), out["image_offsets"].data_ptr(), out["shapes"].data_ptr(),
            out["status"].data_ptr(), torch.cuda.current_stream().cuda_stream), "%s_decode" % kind)
    return out


def _views(res):
    """(list of HWC uint8 views of the buffer, None for a flagged image; status numpy) of a decode_packed result"""
    shapes = res["shapes"].cpu().tolist()
    offs = res["image_offsets"].cpu().tolist()
    status = res["status"].cpu().numpy()
    views = []
    for (h, w), o, s in zip(shapes, offs, status):
        views.append(res["buffer"][o:o + h * w * 3].view(h, w, 3) if s == 0 else None)
    return views, status
