"""Training targets of the DB detector on the device: MakeSegDetectionData (data/processes/make_seg_detection_data.py:21-100)
and MakeBorderMap (make_border_map.py:24-121) for a whole batch, after RandomCropData (csrc/db_targets.cu).

    make_targets(polygons, ignore_tags, size, ...)       -> dict of device tensors, from per-image polygon tensors
    pack(polygons, ignore_tags, capacity)                 -> (polys [capacity, 4, 2], tags [capacity], offsets [N + 1])
    make_targets_packed(polys, tags, offsets, size, ...)  -> the same dict, from packed tensors; never synchronises with the
                                                             host, so it can be captured in a CUDA graph and replayed after
                                                             copying new polygons into the packed tensors

The returned dict holds gt [N,1,H,W], mask, thresh_map and thresh_mask [N,H,W] (float32, as the processes compute them),
polygons (validate_polygons' clipped and reordered quads, in the input dtype), ignore_tags (the updated tags, bool) and
status (int32 bits per polygon, STATUS below).  The shrink and pad restate pyclipper's offset with Clipper 6.4.2's union
clean-up (not pinned against pyclipper; DESIGN §7).  CUDA only; no CPU fallback."""
import numpy as np
import torch

from . import _lib

# per-polygon status bits
STATUS = dict(ignored_in=1, tiny_area=2, small_text=4, shrink_empty=8, shrink_pieces=16, pad_empty=32, pad_pieces=64,
              overflow=128)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def pack(polygons, ignore_tags, capacity=None):
    """Per-image CUDA tensors polygons[n] [k_n, 4, 2] (all float32 or all float64) and ignore_tags[n] [k_n] -> packed
    (polys [capacity, 4, 2], tags uint8 [capacity], offsets int32 [N + 1]) on the same device; capacity defaults to the
    total number of polygons.  Rows past the total are zero."""
    if len(polygons) != len(ignore_tags) or not polygons:
        raise ValueError("db_targets.pack: need one polygon tensor and one tag tensor per image")
    for p, t in zip(polygons, ignore_tags):
        if not (torch.is_tensor(p) and torch.is_tensor(t) and p.is_cuda and t.is_cuda):
            raise NotImplementedError("megreader_b200: db_targets runs on CUDA only (no CPU fallback); pass CUDA tensors")
        if p.dtype not in (torch.float32, torch.float64) or p.dtype != polygons[0].dtype or p.device != polygons[0].device:
            raise RuntimeError("db_targets.pack: polygons must all be float32 or all float64 on one device")
        if p.dim() != 3 or p.shape[1:] != (4, 2) or t.dim() != 1 or t.numel() != p.size(0) or t.device != p.device:
            raise RuntimeError("db_targets.pack: expected polygons [n, 4, 2] and ignore_tags [n], got %s and %s"
                               % (tuple(p.shape), tuple(t.shape)))
    counts = [int(p.size(0)) for p in polygons]
    total = sum(counts)
    capacity = total if capacity is None else int(capacity)
    if capacity < total:
        raise ValueError("db_targets.pack: %d polygons do not fit capacity %d" % (total, capacity))
    dev = polygons[0].device
    polys = torch.zeros((capacity, 4, 2), dtype=polygons[0].dtype, device=dev)
    tags = torch.zeros((capacity,), dtype=torch.uint8, device=dev)
    if total:
        polys[:total] = torch.cat(polygons)
        tags[:total] = torch.cat([t.to(torch.uint8) for t in ignore_tags])
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(counts)]), dtype=torch.int32).to(dev)
    return polys, tags, offsets


def make_targets_packed(polys, tags, offsets, size, shrink_ratio=0.4, min_text_size=8, thresh_min=0.3, thresh_max=0.7):
    """The targets of N = offsets.numel() - 1 images of size (H, W) from packed polygons (see pack); no host
    synchronisation.  Workspace: about 120 KB per polygon slot at 640 x 640."""
    for name, t in (("polygons", polys), ("ignore_tags", tags), ("offsets", offsets)):
        if not (torch.is_tensor(t) and t.is_cuda):
            raise NotImplementedError("megreader_b200: db_targets runs on CUDA only (no CPU fallback); %s is not a CUDA tensor" % name)
    if polys.dtype not in (torch.float32, torch.float64) or polys.dim() != 3 or polys.shape[1:] != (4, 2):
        raise RuntimeError("db_targets: polygons must be float32 or float64 [capacity, 4, 2], got %s %s" % (polys.dtype, tuple(polys.shape)))
    cap = polys.size(0)
    if tags.dtype != torch.uint8 or tags.shape != (cap,) or offsets.dtype != torch.int32 or offsets.dim() != 1 or offsets.numel() < 2:
        raise RuntimeError("db_targets: ignore_tags must be uint8 [capacity] and offsets int32 [N + 1]")
    if tags.device != polys.device or offsets.device != polys.device:
        raise RuntimeError("db_targets: polygons, ignore_tags and offsets must be on one device")
    polys, tags, offsets = polys.contiguous(), tags.contiguous(), offsets.contiguous()
    N = offsets.numel() - 1
    H, W = int(size[0]), int(size[1])
    dev = polys.device
    L = _lib.lib()
    nbytes = int(L.mr_db_targets_workspace_bytes(N, H, W, cap))
    if nbytes <= 0:
        raise RuntimeError("db_targets: unsupported sizes N=%d, H=%d, W=%d, capacity=%d" % (N, H, W, cap))
    f32 = dict(dtype=torch.float32, device=dev)
    out = dict(gt=torch.empty((N, 1, H, W), **f32), mask=torch.empty((N, H, W), **f32), thresh_map=torch.empty((N, H, W), **f32),
               thresh_mask=torch.empty((N, H, W), **f32), polygons=torch.empty_like(polys),
               ignore_tags=torch.empty((cap,), dtype=torch.uint8, device=dev), status=torch.empty((cap,), dtype=torch.int32, device=dev))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    shrink_k = float(1 - np.power(shrink_ratio, 2))
    with torch.cuda.device(dev):
        _lib.check(L.mr_db_targets(polys.data_ptr(), int(polys.dtype == torch.float64), tags.data_ptr(), offsets.data_ptr(), N, H, W,
                                   cap, shrink_k, float(min_text_size), float(np.float32(thresh_max - thresh_min)),
                                   float(np.float32(thresh_min)), ws.data_ptr(), nbytes, out["gt"].data_ptr(), out["mask"].data_ptr(),
                                   out["thresh_map"].data_ptr(), out["thresh_mask"].data_ptr(), out["polygons"].data_ptr(),
                                   out["ignore_tags"].data_ptr(), out["status"].data_ptr(), _stream()), "db_targets")
    out["workspace"] = ws
    return out


def make_targets(polygons, ignore_tags, size, shrink_ratio=0.4, min_text_size=8, thresh_min=0.3, thresh_max=0.7):
    """MakeSegDetectionData + MakeBorderMap for a batch: polygons[n] [k_n, 4, 2] float32 or float64 and ignore_tags[n] [k_n]
    CUDA tensors, size (H, W) -> dict(gt, mask, thresh_map, thresh_mask, polygons (list per image), ignore_tags (list of
    bool tensors per image), status (list of int32 tensors per image))."""
    polys, tags, offsets = pack(polygons, ignore_tags)
    out = make_targets_packed(polys, tags, offsets, size, shrink_ratio, min_text_size, thresh_min, thresh_max)
    counts = [int(p.size(0)) for p in polygons]
    out.pop("workspace")
    out["polygons"] = list(torch.split(out["polygons"], counts))
    out["ignore_tags"] = [t.bool() for t in torch.split(out["ignore_tags"], counts)]
    out["status"] = list(torch.split(out["status"], counts))
    return out
