"""Text crops for recognition on the device: ImageCropper.crop (data/crop_file_dataset.py:85-124) for every quad of a batch
(csrc/text_crop.cu).

    crop_quads_packed(buffer, image_offsets, shapes, quads, count, ...)  -> dict(image [capacity, 3, H, W], owner [capacity, 2],
                                                                             total [1], status [N]); never synchronises with
                                                                             the host, so it can be captured in a CUDA graph
    crop_quads(images, quads, counts, ...)                               -> the same from a list of HWC images
    ImageCropper(image_size=(64, 512), mode="resize").crop(image, poly)  -> the reference's HWC float32 crop

Each quad goes through cv2.minAreaRect with the reference's angle rule and cv2.boxPoints, a cv2.warpPerspective of the source
into an int(w) x int(h) crop (the source's size when a side truncates to 0), the turn of tall crops, ResizeImage ("resize" or
"pad") and NormalizeImage -- without the crop ever being stored.  CUDA only; no CPU fallback."""
import torch

from . import _lib, db_batch

RGB_MEAN = (122.67891434, 116.66876762, 104.00698793)      # crop_file_dataset.py (applied in stored channel order)
MODES = ("resize", "pad")

# per-image status bits
STATUS = dict(bad_shape=1, bad_pixels=2, bad_count=4, overflow=8, zero_side=16, crop_too_large=32)


def _cuda(t, name):
    if not (torch.is_tensor(t) and t.is_cuda):
        raise NotImplementedError("megreader_b200: text_crop runs on CUDA only (no CPU fallback); %s is not a CUDA tensor" % name)


def crop_quads_packed(buffer, image_offsets, shapes, quads, count, image_size=(64, 512), mode="resize", capacity=None):
    """Crops of every quad of N images packed by db_batch.pack_images (HWC uint8 or float32, BGR as decoded).

    quads / count: boxes_from_maps' (boxes int32 [N, K, 4, 2], count int32 [N]), or packed quads [P, 4, 2] (int32 or
    float32) with offsets int32 [N + 1] as db_targets.pack returns them.  Rows are the quads in (image, quad) order; capacity
    defaults to N * K (or P).  Returns image float32 [capacity, 3, image_size[0], image_size[1]] (rows >= total are not
    written), owner int32 [capacity, 2] ((image, quad) of each row, -1 past the total), total int32 [1] (the number of quads,
    which may exceed capacity) and status int32 [N] (STATUS bits: overflow when some of the image's quads found no row,
    zero_side when one of its crops took the source's size).  No host synchronisation."""
    if mode not in MODES:
        raise ValueError("text_crop: mode must be 'resize' or 'pad' (fixed-size outputs), got %r" % (mode,))
    for name, t in (("buffer", buffer), ("image_offsets", image_offsets), ("shapes", shapes), ("quads", quads), ("count", count)):
        _cuda(t, name)
    if buffer.dtype not in (torch.uint8, torch.float32) or buffer.dim() != 1:
        raise RuntimeError("text_crop: the image buffer must be flat uint8 or float32")
    N = image_offsets.numel()
    if image_offsets.dtype != torch.int64 or image_offsets.dim() != 1 or N < 1 or shapes.dtype != torch.int32 or shapes.shape != (N, 2):
        raise RuntimeError("text_crop: image_offsets must be int64 [N] and shapes int32 [N, 2]")
    if quads.dtype not in (torch.int32, torch.float32) or quads.dim() not in (3, 4) or quads.shape[-2:] != (4, 2):
        raise RuntimeError("text_crop: quads must be int32 or float32 [N, K, 4, 2] or [P, 4, 2], got %s %s"
                           % (quads.dtype, tuple(quads.shape)))
    if quads.dim() == 4:
        K = quads.size(1)
        if quads.size(0) != N or count.dtype != torch.int32 or count.shape != (N,):
            raise RuntimeError("text_crop: quads [N, K, 4, 2] need count int32 [N]")
        cap = N * K if capacity is None else int(capacity)
        if K == 0:                       # no candidates: a zero quad per image keeps the pointer valid; a count > 0 is refused
            quads = quads.new_zeros((N, 1, 4, 2))
            count = torch.where(count > 0, -1, count)
            K = 1
        rows = N * K
    else:
        K, rows = 0, quads.size(0)
        if count.dtype != torch.int32 or count.shape != (N + 1,):
            raise RuntimeError("text_crop: packed quads [P, 4, 2] need offsets int32 [N + 1]")
        cap = rows if capacity is None else int(capacity)
    dev = buffer.device
    if any(t.device != dev for t in (image_offsets, shapes, quads, count)):
        raise RuntimeError("text_crop: every tensor must be on one device")
    buffer, image_offsets, shapes = buffer.contiguous(), image_offsets.contiguous(), shapes.contiguous()
    quads, count = quads.contiguous(), count.contiguous()
    out_h, out_w = int(image_size[0]), int(image_size[1])
    L = _lib.lib()
    nbytes = int(L.mr_text_crop_workspace_bytes(N, cap))
    if nbytes <= 0:
        raise RuntimeError("text_crop: unsupported sizes N=%d, capacity=%d" % (N, cap))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out = dict(image=torch.empty((cap, 3, out_h, out_w), dtype=torch.float32, device=dev),
               owner=torch.empty((cap, 2), dtype=torch.int32, device=dev),
               total=torch.empty((1,), dtype=torch.int32, device=dev),
               status=torch.empty((N,), dtype=torch.int32, device=dev))
    with torch.cuda.device(dev):
        _lib.check(L.mr_text_crop(buffer.data_ptr(), int(buffer.dtype == torch.float32), buffer.numel(), image_offsets.data_ptr(),
                                  shapes.data_ptr(), N, quads.data_ptr(), int(quads.dtype == torch.float32), rows, K,
                                  count.data_ptr(), cap, MODES.index(mode), out_h, out_w, *[float(m) for m in RGB_MEAN],
                                  ws.data_ptr(), nbytes, out["image"].data_ptr(), out["owner"].data_ptr(), out["total"].data_ptr(),
                                  out["status"].data_ptr(), torch.cuda.current_stream().cuda_stream), "text_crop")
    out["workspace"] = ws
    return out


def crop_quads(images, quads, counts=None, image_size=(64, 512), mode="resize", capacity=None):
    """images: per-image HWC CUDA tensors (all uint8 or all float32); quads: boxes_from_maps' [N, K, 4, 2] with counts [N],
    or a list of per-image [k_n, 4, 2] tensors (counts None).  Returns crop_quads_packed's dict."""
    buffer, image_offsets, shapes = db_batch.pack_images(images)
    if isinstance(quads, (list, tuple)):
        if len(quads) != len(images):
            raise ValueError("text_crop: need one quad tensor per image")
        for q in quads:
            _cuda(q, "a quad tensor")
        dtype = torch.float32 if any(q.dtype != torch.int32 for q in quads) else torch.int32
        packed = torch.cat([q.reshape(-1, 4, 2).to(dtype) for q in quads]) if quads else None
        sizes = [int(q.reshape(-1, 4, 2).size(0)) for q in quads]
        offs = [0]
        for s in sizes:
            offs.append(offs[-1] + s)
        counts = torch.tensor(offs, dtype=torch.int32).to(buffer.device)
        quads = packed
    elif counts is None:
        raise ValueError("text_crop: quads [N, K, 4, 2] need counts")
    return crop_quads_packed(buffer, image_offsets, shapes, quads, counts, image_size, mode, capacity)


class ImageCropper:
    """data/crop_file_dataset.py's ImageCropper: crop(image, poly) of one HWC CUDA image (uint8 or float32) and one quad
    [4, 2] -> the reference's HWC float32 [image_size[0], image_size[1], 3] crop, as a CUDA tensor."""

    def __init__(self, image_size=(64, 512), mode="resize"):
        if mode not in MODES:
            raise ValueError("ImageCropper: mode %r is not supported (fixed-size modes: %s)" % (mode, ", ".join(MODES)))
        self.image_size = (int(image_size[0]), int(image_size[1]))
        self.mode = mode

    def crop(self, image, poly):
        _cuda(image, "image")
        poly = torch.as_tensor(poly, device=image.device)
        poly = poly.to(torch.int32 if poly.dtype == torch.int32 else torch.float32).reshape(1, 4, 2)
        out = crop_quads([image], [poly], image_size=self.image_size, mode=self.mode)
        return out["image"][0].permute(1, 2, 0).contiguous()
