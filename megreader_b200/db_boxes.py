"""The DB detector's SegDetectorRepresenter (structure/representers/seg_detector_representer.py:10-168) on the device
(csrc/db_boxes.cu).

    boxes_from_maps(binary, dest, thresh, box_thresh, max_candidates, dest_sizes)  -> (boxes, scores, count), device tensors
    SegDetectorRepresenter(thresh, box_thresh, max_candidates, resize, dest).represent(batch, pred) -> (boxes_batch, pred)

and the two stages the first one is made of, for callers that want the contours or the candidates themselves:

    find_contours(dest, thresh, max_candidates)             -> (points, offsets, count, total)
    box_candidates(binary, points, offsets, count)          -> (boxes, ssides, scores)
    contour_lists(points, offsets, count)                   -> per image, the list cv2.findContours(...)[:max_candidates] returns

`boxes_from_maps` is boxes_from_bitmap (:63-115) for a whole batch: the contours of `dest > thresh` exactly as
cv2.findContours(RETR_LIST, CHAIN_APPROX_NONE) gives them, truncated to max_candidates, and for every candidate
get_mini_boxes, `sside < 3`, box_score_fast, `box_thresh > score`, the unclip, the second get_mini_boxes, `sside < 5` and the
rescale, the survivors compacted in candidate order.  It never synchronises with the host, so it can be captured in a CUDA
graph; `represent` adds the one copy to the host.  The unclip restates Clipper's round offset without its final union clean-up
(not pinned against pyclipper; DESIGN §7).  CUDA only; no CPU fallback."""
import numpy as np
import torch

from . import _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def find_contours(dest, thresh=0.3, max_candidates=100, point_capacity=None):
    """dest [N,1,H,W] (or [N,H,W]) fp32 on CUDA -> (points int32 [N,P,2] (x, y), offsets int32 [N,max_candidates+1],
    count int32 [N] = min(total, max_candidates), total int32 [N] = contours in the image).  Contour c < count[n] of image n is
    points[n, offsets[n,c]:offsets[n,c+1]].  P = point_capacity, by default 4 * H * W (32 bytes per pixel; real contour sets use
    a small fraction of it, and a tighter capacity is safe because overflow is reported, not silent): points past it are not
    written, the offsets still count them, contour_lists raises and box_candidates marks those contours with sside -1.  The
    exact size would need a host read of the counted lengths, which would break graph capture."""
    if not dest.is_cuda:
        raise NotImplementedError("megreader_b200: find_contours runs on CUDA only (no CPU fallback)")
    if dest.dtype != torch.float32 or dest.dim() not in (3, 4) or (dest.dim() == 4 and dest.size(1) != 1):
        raise RuntimeError("find_contours: expected an fp32 map [N,1,H,W] or [N,H,W], got %s %s" % (dest.dtype, tuple(dest.shape)))
    N, H, W = dest.size(0), dest.size(-2), dest.size(-1)
    maxc = int(max_candidates)
    if maxc < 0:
        raise ValueError("find_contours: max_candidates must be >= 0, got %d" % maxc)
    cap = 4 * H * W if point_capacity is None else int(point_capacity)
    dest = dest.contiguous()
    dev = dest.device
    L = _lib.lib()
    i32 = dict(dtype=torch.int32, device=dev)
    points = torch.empty((N, cap, 2), **i32)
    offsets = torch.empty((N, maxc + 1), **i32)
    count = torch.empty((N,), **i32)
    total = torch.empty((N,), **i32)
    if N == 0:
        return points, offsets, count, total
    nbytes = int(L.mr_db_contours_workspace_bytes(N, H, W, maxc))
    if nbytes <= 0:
        raise RuntimeError("find_contours: unsupported map size %s" % (tuple(dest.shape),))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.mr_db_contours_f32(dest.data_ptr(), N, H, W, float(thresh), maxc, ws.data_ptr(), nbytes, points.data_ptr(),
                                        cap, offsets.data_ptr(), count.data_ptr(), total.data_ptr(), _stream()), "db_contours")
    return points, offsets, count, total


def box_candidates(binary, points, offsets, count):
    """binary [N,1,H,W] (or [N,H,W]) fp32, the score map, and the outputs of find_contours -> (boxes fp32 [N, max_candidates, 4, 2],
    ssides fp32 [N, max_candidates], scores fp64 [N, max_candidates]): get_mini_boxes' corners and min(width, height) for every
    kept contour, and box_score_fast where sside >= 3 (0 elsewhere); zero past count[n]; sside -1 for a contour whose points did
    not fit the point capacity."""
    if not (binary.is_cuda and points.is_cuda and offsets.is_cuda and count.is_cuda):
        raise NotImplementedError("megreader_b200: box_candidates runs on CUDA only (no CPU fallback)")
    for name, t, dim in (("points", points, 3), ("offsets", offsets, 2), ("count", count, 1)):
        if t.dtype != torch.int32 or t.dim() != dim or not t.is_contiguous() or t.device != binary.device:
            raise RuntimeError("box_candidates: %s must be a contiguous int32 tensor of %d dimensions on %s (find_contours' "
                               "output), got %s %s on %s" % (name, dim, binary.device, t.dtype, tuple(t.shape), t.device))
    N, cap = points.size(0), points.size(1)
    maxc = offsets.size(1) - 1
    if points.size(2) != 2 or offsets.size(0) != N or count.size(0) != N:
        raise RuntimeError("box_candidates: points [N,P,2], offsets [N,max_candidates+1] and count [N] do not match")
    if binary.dtype != torch.float32 or binary.dim() not in (3, 4) or binary.size(0) != N or (binary.dim() == 4 and binary.size(1) != 1):
        raise RuntimeError("box_candidates: expected an fp32 score map [N,1,H,W] or [N,H,W] with N = %d, got %s %s"
                           % (N, binary.dtype, tuple(binary.shape)))
    H, W = binary.size(-2), binary.size(-1)
    binary = binary.contiguous()
    dev = points.device
    boxes = torch.zeros((N, maxc, 4, 2), dtype=torch.float32, device=dev)
    ssides = torch.zeros((N, maxc), dtype=torch.float32, device=dev)
    scores = torch.zeros((N, maxc), dtype=torch.float64, device=dev)
    if N == 0 or maxc == 0:
        return boxes, ssides, scores
    L = _lib.lib()
    nbytes = int(L.mr_db_box_candidates_workspace_bytes(N, maxc, cap))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.mr_db_box_candidates_f32(points.data_ptr(), cap, offsets.data_ptr(), count.data_ptr(), binary.data_ptr(), N, H,
                                              W, maxc, ws.data_ptr(), nbytes, boxes.data_ptr(), ssides.data_ptr(),
                                              scores.data_ptr(), _stream()), "db_box_candidates")
    return boxes, ssides, scores


def contour_lists(points, offsets, count):
    """The outputs of find_contours -> per image, a list of int32 arrays [k,1,2] as cv2.findContours returns them."""
    count = count.cpu().numpy()
    offsets = offsets.cpu().numpy()
    ends = offsets[np.arange(len(count)), count]
    if (ends > points.size(1)).any():
        raise RuntimeError("find_contours: %d contour points do not fit the point capacity %d" % (int(ends.max()), points.size(1)))
    keep = int(ends.max()) if len(count) else 0
    pts = points[:, :keep].cpu().numpy()
    return [[pts[n, offsets[n, c]:offsets[n, c + 1]].reshape(-1, 1, 2) for c in range(count[n])] for n in range(len(count))]


def boxes_from_maps(binary, dest=None, thresh=0.3, box_thresh=0.7, max_candidates=100, dest_sizes=None):
    """binary (the score map, pred['binary']) and dest (the bitmap source: binary, thresh or thresh_binary; None = binary),
    [N,1,H,W] fp32 on CUDA; dest_sizes int [N,2] of (height, width) to rescale to, or None for (H, W) -> (boxes int32
    [N, max_candidates, 4, 2] (x, y), scores fp32 [N, max_candidates], count int32 [N]); entries past count[n] are zero.
    The workspace is about 136 bytes per map pixel (find_contours' 4 * H * W point capacity and the candidate scratch)."""
    dest = binary if dest is None else dest
    if not (binary.is_cuda and dest.is_cuda):
        raise NotImplementedError("megreader_b200: boxes_from_maps runs on CUDA only (no CPU fallback)")
    for name, t in (("binary", binary), ("dest", dest)):
        if t.dtype != torch.float32 or t.dim() not in (3, 4) or (t.dim() == 4 and t.size(1) != 1):
            raise RuntimeError("boxes_from_maps: %s must be an fp32 map [N,1,H,W] or [N,H,W], got %s %s"
                               % (name, t.dtype, tuple(t.shape)))
    N, H, W = binary.size(0), binary.size(-2), binary.size(-1)
    if (dest.size(0), dest.size(-2), dest.size(-1)) != (N, H, W) or dest.device != binary.device:
        raise RuntimeError("boxes_from_maps: dest %s does not match binary %s" % (tuple(dest.shape), tuple(binary.shape)))
    maxc = int(max_candidates)
    if maxc < 0:
        raise ValueError("boxes_from_maps: max_candidates must be >= 0, got %d" % maxc)
    dev = binary.device
    binary, dest = binary.contiguous(), dest.contiguous()
    if dest_sizes is not None:
        dest_sizes = torch.as_tensor(dest_sizes).to(device=dev, dtype=torch.int32).reshape(N, 2).contiguous()
    boxes = torch.empty((N, maxc, 4, 2), dtype=torch.int32, device=dev)
    scores = torch.empty((N, maxc), dtype=torch.float32, device=dev)
    count = torch.empty((N,), dtype=torch.int32, device=dev)
    if N == 0:
        return boxes, scores, count
    L = _lib.lib()
    nbytes = int(L.mr_db_boxes_workspace_bytes(N, H, W, maxc))
    if nbytes <= 0:
        raise RuntimeError("boxes_from_maps: unsupported batch / map size %s" % (tuple(binary.shape),))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.mr_db_boxes_f32(binary.data_ptr(), dest.data_ptr(), N, H, W, float(thresh), float(box_thresh), maxc,
                                     dest_sizes.data_ptr() if dest_sizes is not None else None, ws.data_ptr(), nbytes,
                                     boxes.data_ptr(), scores.data_ptr(), count.data_ptr(), _stream()), "db_boxes")
    return boxes, scores, count


class SegDetectorRepresenter:
    """The reference's SegDetectorRepresenter (seg_detector_representer.py:10-58) with its defaults; represent() returns the
    reference's structure -- per image a list of boxes [[x, y]] * 4 (floats, as box.tolist() gives them) -- and pred.  The one
    copy to the host is the final one.  Debug drawing is not reproduced."""

    def __init__(self, thresh=0.3, box_thresh=0.7, max_candidates=100, resize=False, dest='binary'):
        self.thresh, self.box_thresh, self.max_candidates, self.resize, self.dest = thresh, box_thresh, max_candidates, resize, dest
        self.min_size = 3

    def represent(self, batch, _pred):
        sizes = None
        if self.resize:
            sizes = torch.as_tensor([[int(h), int(w)] for h, w in batch['shape']], dtype=torch.int32)
        boxes, _, count = boxes_from_maps(_pred['binary'], _pred[self.dest], self.thresh, self.box_thresh, self.max_candidates,
                                          sizes)
        boxes, count = boxes.cpu().numpy(), count.cpu().numpy()
        return [boxes[n, :count[n]].astype(np.float64).tolist() for n in range(len(count))], _pred

