"""The DB detector's input batch on the device: seg_detector_db.yaml's data processes before the targets
(AugmentDetectionData, RandomCropData, MakeICDARData, NormalizeImage) for a whole batch (csrc/db_batch.cu).

    pack_images(images)                      -> (buffer, image_offsets int64 [N], shapes int32 [N, 2]) from HWC uint8 or float32
    draws(N, generator, max_tries)           -> [N, 3 + 8 * max_tries] float32 uniform draws on the device
    train_batch_packed(...)                  -> dict of device tensors: the augmented, cropped, normalised images and the
    validate_batch_packed(...)                  kept quads packed for db_targets.make_targets_packed; never synchronises with
                                                the host, so it can be captured in a CUDA graph
    train_batch(images, polygons, ignore_tags, generator)   -> what the training step consumes (image, gt, mask, thresh_map,
                                                               thresh_mask)
    validate_batch(images, polygons, ignore_tags)           -> what ICDARCollectFN returns (image, polygons, ignore_tags, shape
                                                               and the targets)

Training restates imgaug's Sequential([Fliplr(0.5), Affine(rotate=(-10, 10)), Resize((0.5, 3.0))]) (after imgaug 0.4.0, cv2
backend; DESIGN §7) and RandomCropData exactly, from the draws: flip when draws[:, 0] < flip_p, the angle
rotate[0] + draws[:, 1] * (rotate[1] - rotate[0]), the scale likewise from draws[:, 2], and crop_area's np.random.choice picks
axis[min(floor(u * len), len - 1)] from draws[:, 3 + 4 * (round * max_tries + try) + (0, 1 for x; 2, 3 for y)].  The random
streams are the device's: the batches are statistically, not sample for sample, those of the reference's loader.  Only this
augmenter chain and quads are supported.  CUDA only; no CPU fallback."""
import torch

from . import _lib, db_targets

RGB_MEAN = (122.67891434, 116.66876762, 104.00698793)      # normalize_image.py (applied in stored channel order)

# per-image status bits
STATUS = dict(bad_shape=1, bad_pixels=2, bad_offsets=4)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cuda(t, name):
    if not (torch.is_tensor(t) and t.is_cuda):
        raise NotImplementedError("megreader_b200: db_batch runs on CUDA only (no CPU fallback); %s is not a CUDA tensor" % name)


def draws_per_image(max_tries=10):
    return 3 + 8 * int(max_tries)


def draws(N, generator=None, max_tries=10, device=None):
    """[N, 3 + 8 * max_tries] float32 uniform [0, 1) draws on the device (torch.rand: graph capture records it)."""
    dev = generator.device if generator is not None else (device or torch.device("cuda", torch.cuda.current_device()))
    return torch.rand((int(N), draws_per_image(max_tries)), generator=generator, device=dev, dtype=torch.float32)


def pack_images(images):
    """Per-image HWC CUDA tensors (all uint8 or all float32, 3 channels) -> (buffer, image_offsets int64 [N] in elements,
    shapes int32 [N, 2] as (h, w)), all on the images' device."""
    if not images:
        raise ValueError("db_batch.pack_images: need at least one image")
    for im in images:
        _cuda(im, "an image")
        if im.dtype not in (torch.uint8, torch.float32) or im.dtype != images[0].dtype or im.device != images[0].device:
            raise RuntimeError("db_batch.pack_images: images must all be uint8 or all float32 on one device")
        if im.dim() != 3 or im.size(2) != 3:
            raise RuntimeError("db_batch.pack_images: expected HWC images with 3 channels, got %s" % (tuple(im.shape),))
    dev = images[0].device
    sizes = [im.numel() for im in images]
    offs = [0]
    for s in sizes[:-1]:
        offs.append(offs[-1] + s)
    buffer = torch.cat([im.reshape(-1) for im in images])
    image_offsets = torch.tensor(offs, dtype=torch.int64).to(dev)
    shapes = torch.tensor([[im.size(0), im.size(1)] for im in images], dtype=torch.int32).to(dev)
    return buffer, image_offsets, shapes


def _call(mode, buffer, image_offsets, shapes, max_h, max_w, polys, tags, offsets, u, out_h, out_w, max_tries, min_crop_side_ratio,
          rotate, scale, flip_p):
    for name, t in (("buffer", buffer), ("image_offsets", image_offsets), ("shapes", shapes), ("polygons", polys),
                    ("ignore_tags", tags), ("offsets", offsets)):
        _cuda(t, name)
    if buffer.dtype not in (torch.uint8, torch.float32) or buffer.dim() != 1:
        raise RuntimeError("db_batch: the image buffer must be flat uint8 or float32")
    N = image_offsets.numel()
    if image_offsets.dtype != torch.int64 or image_offsets.dim() != 1 or N < 1 or shapes.dtype != torch.int32 or shapes.shape != (N, 2):
        raise RuntimeError("db_batch: image_offsets must be int64 [N] and shapes int32 [N, 2]")
    if polys.dtype not in (torch.float32, torch.float64) or polys.dim() != 3 or polys.shape[1:] != (4, 2):
        raise RuntimeError("db_batch: polygons must be float32 or float64 [capacity, 4, 2], got %s %s" % (polys.dtype, tuple(polys.shape)))
    cap = polys.size(0)
    if tags.dtype != torch.uint8 or tags.shape != (cap,) or offsets.dtype != torch.int32 or offsets.shape != (N + 1,):
        raise RuntimeError("db_batch: ignore_tags must be uint8 [capacity] and offsets int32 [N + 1]")
    if mode == 0:
        _cuda(u, "draws")
        if u.dtype != torch.float32 or u.dim() != 2 or u.size(0) != N or u.size(1) < draws_per_image(max_tries):
            raise RuntimeError("db_batch: draws must be float32 [N, >= %d]" % draws_per_image(max_tries))
        u = u.contiguous()
    dev = buffer.device
    if any(t.device != dev for t in (image_offsets, shapes, polys, tags, offsets)) or (mode == 0 and u.device != dev):
        raise RuntimeError("db_batch: every tensor must be on one device")
    buffer, image_offsets, shapes = buffer.contiguous(), image_offsets.contiguous(), shapes.contiguous()
    polys, tags, offsets = polys.contiguous(), tags.contiguous(), offsets.contiguous()
    L = _lib.lib()
    nbytes = int(L.mr_db_batch_workspace_bytes(N, int(max_h), int(max_w), cap))
    if nbytes <= 0:
        raise RuntimeError("db_batch: unsupported sizes N=%d, max_h=%d, max_w=%d, capacity=%d" % (N, max_h, max_w, cap))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out = dict(image=torch.empty((N, 3, out_h, out_w), dtype=torch.float32, device=dev),
               polygons=torch.empty((cap, 4, 2), dtype=torch.float64, device=dev),
               ignore_tags=torch.empty((cap,), dtype=torch.uint8, device=dev),
               offsets=torch.empty((N + 1,), dtype=torch.int32, device=dev),
               shape=torch.empty((N, 2), dtype=torch.int32, device=dev),
               crop=torch.empty((N, 4), dtype=torch.int32, device=dev),
               scale=torch.empty((N,), dtype=torch.float64, device=dev),
               status=torch.empty((N,), dtype=torch.int32, device=dev))
    with torch.cuda.device(dev):
        _lib.check(L.mr_db_batch(buffer.data_ptr(), int(buffer.dtype == torch.float32), buffer.numel(), image_offsets.data_ptr(),
                                 shapes.data_ptr(), N, int(max_h), int(max_w), polys.data_ptr(), int(polys.dtype == torch.float64),
                                 tags.data_ptr(), offsets.data_ptr(), cap, u.data_ptr() if mode == 0 else None,
                                 u.size(1) if mode == 0 else 0, mode, int(out_h), int(out_w), int(max_tries),
                                 float(min_crop_side_ratio), float(flip_p), float(rotate[0]), float(rotate[1]), float(scale[0]),
                                 float(scale[1]), *[float(m) for m in RGB_MEAN], ws.data_ptr(), nbytes, out["image"].data_ptr(),
                                 out["polygons"].data_ptr(), out["ignore_tags"].data_ptr(), out["offsets"].data_ptr(),
                                 out["shape"].data_ptr(), out["crop"].data_ptr(), out["scale"].data_ptr(), out["status"].data_ptr(),
                                 _stream()), "db_batch")
    out["workspace"] = ws
    return out


def train_batch_packed(buffer, image_offsets, shapes, max_h, max_w, polys, tags, offsets, u, size=(640, 640), max_tries=10,
                       min_crop_side_ratio=0.1, rotate=(-10, 10), scale=(0.5, 3.0), flip_p=0.5):
    """AugmentDetectionData + RandomCropData(size = (width, height)) + MakeICDARData + NormalizeImage for N images packed by
    pack_images (each at most max_h x max_w) with quads packed by db_targets.pack, from the draws u (see draws).  Returns
    image [N, 3, size[1], size[0]] float32, polygons float64 [capacity, 4, 2] with ignore_tags uint8 and offsets int32 [N + 1]
    (the kept quads, as make_targets_packed takes them), shape [N, 2] (the input's (h, w)), crop [N, 4] (x, y, w, h in the
    resized image), scale [N] float64 and status [N] (STATUS bits; such an image has no quads and a zero canvas).  No host
    synchronisation.  Workspace: about 12 bytes per pixel of N x max_h x max_w."""
    return _call(0, buffer, image_offsets, shapes, max_h, max_w, polys, tags, offsets, u, int(size[1]), int(size[0]), max_tries,
                 min_crop_side_ratio, rotate, scale, flip_p)


def validate_batch_packed(buffer, image_offsets, shapes, max_h, max_w, polys, tags, offsets, size=(576, 1024)):
    """AugmentDetectionData([Resize({'width': size[1], 'height': size[0]})]) + MakeICDARData + NormalizeImage: the same
    outputs as train_batch_packed with image [N, 3, size[0], size[1]], every quad kept, crop the whole resized image and
    scale 1.  No host synchronisation."""
    return _call(1, buffer, image_offsets, shapes, max_h, max_w, polys, tags, offsets, None, int(size[0]), int(size[1]), 1, 0.,
                 (0., 0.), (1., 1.), 0.)


def _pack_all(images, polygons, ignore_tags):
    if len(images) != len(polygons):
        raise ValueError("db_batch: need one polygon tensor per image")
    buffer, image_offsets, shapes = pack_images(images)
    polys, tags, offsets = db_targets.pack(polygons, ignore_tags)
    max_h = max(int(im.size(0)) for im in images)
    max_w = max(int(im.size(1)) for im in images)
    return buffer, image_offsets, shapes, max_h, max_w, polys, tags, offsets


def _checked(out):
    bad = out["status"].nonzero().flatten().tolist()
    if bad:
        raise RuntimeError("db_batch: images %s were refused (status %s)" % (bad, out["status"][bad].tolist()))


def train_batch(images, polygons, ignore_tags, generator=None, size=(640, 640), max_tries=10, min_crop_side_ratio=0.1,
                rotate=(-10, 10), scale=(0.5, 3.0), flip_p=0.5, shrink_ratio=0.4, min_text_size=8, thresh_min=0.3, thresh_max=0.7):
    """The training batch of seg_detector_db.yaml after FilterKeys: images[n] HWC uint8 or float32 CUDA tensors (BGR as
    cv2.imdecode gives them), polygons[n] [k_n, 4, 2] and ignore_tags[n] [k_n] -> dict(image [N, 3, H, W], gt [N, 1, H, W],
    mask, thresh_map, thresh_mask [N, H, W])."""
    args = _pack_all(images, polygons, ignore_tags)
    u = draws(len(images), generator, max_tries, device=args[0].device)
    out = train_batch_packed(*args, u, size, max_tries, min_crop_side_ratio, rotate, scale, flip_p)
    _checked(out)
    t = db_targets.make_targets_packed(out["polygons"], out["ignore_tags"], out["offsets"], (int(size[1]), int(size[0])),
                                       shrink_ratio, min_text_size, thresh_min, thresh_max)
    return dict(image=out["image"], gt=t["gt"], mask=t["mask"], thresh_map=t["thresh_map"], thresh_mask=t["thresh_mask"])


def validate_batch(images, polygons, ignore_tags, size=(576, 1024), shrink_ratio=0.4, min_text_size=8, thresh_min=0.3,
                   thresh_max=0.7):
    """The validation batch as ICDARCollectFN collates it: dict(image [N, 3, H, W], polygons (list of float64 [k_n, 4, 2]),
    ignore_tags (list of bool [k_n]), shape [N, 2] (the input sizes), gt, mask, thresh_map, thresh_mask), on the device."""
    args = _pack_all(images, polygons, ignore_tags)
    out = validate_batch_packed(*args, size)
    _checked(out)
    t = db_targets.make_targets_packed(out["polygons"], out["ignore_tags"], out["offsets"], size, shrink_ratio, min_text_size,
                                       thresh_min, thresh_max)
    counts = out["offsets"].diff().tolist()
    total = sum(counts)
    # MakeSegDetectionData leaves its validated quads and updated tags in the sample
    return dict(image=out["image"], polygons=list(torch.split(t["polygons"][:total], counts)),
                ignore_tags=[x.bool() for x in torch.split(t["ignore_tags"][:total], counts)], shape=out["shape"],
                gt=t["gt"], mask=t["mask"], thresh_map=t["thresh_map"], thresh_mask=t["thresh_mask"])
