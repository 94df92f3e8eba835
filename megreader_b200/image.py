"""Decoding of batches that mix JPEG and PNG files on the device (csrc/png.cu, mr_image_decode): the replacement of
cv2.imread(path, cv2.IMREAD_COLOR) / cv2.imdecode(buf, cv2.IMREAD_COLOR) in the datasets' loaders.  Each file is decoded by
the decoder whose signature it carries (megreader_b200.jpeg, megreader_b200.png), a file with neither is flagged
(STATUS bad_header); every image equals what the single-format call gives for it.

    decode_packed(data, offsets, max_h, max_w, cap)     -> dict(buffer, image_offsets, shapes, status), graph-capturable
    decode(blobs)                                       -> (list of HWC uint8 CUDA views, status int32 [N] on the host)
"""
from . import _lib, png
from .jpeg import MAX_SIDE, STATUS, _header_pixels, pack_bytes  # noqa: F401
from .png import _decode_packed_with, _views


def workspace_bytes(n, byte_capacity, pixel_capacity):
    return int(_lib.lib().mr_image_workspace_bytes(n, byte_capacity, pixel_capacity))


def decode_packed(data, offsets, max_h, max_w, pixel_capacity, out=None):
    """as jpeg.decode_packed, for JPEG and PNG files in one batch"""
    return _decode_packed_with("image", data, offsets, max_h, max_w, pixel_capacity, out)


def decode(blobs, max_h=MAX_SIDE, max_w=MAX_SIDE, pixel_capacity=None, device=None):
    """the one-call form of cv2.imdecode(buf, cv2.IMREAD_COLOR) for a list of JPEG or PNG byte strings; pixel_capacity
    defaults to the sum over the SOF / IHDR headers"""
    data, offsets = pack_bytes(blobs, device)
    if pixel_capacity is None:
        pixel_capacity = sum(png.header_pixels(b) or _header_pixels(b) for b in blobs)
    return _views(decode_packed(data, offsets, max_h, max_w, max(int(pixel_capacity), 1)))
