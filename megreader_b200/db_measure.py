"""Validation measure of the DB detector on the device: QuadMeasurer (structure/measurers/quad_measurer.py) and the
DetectionIoUEvaluator it calls (concern/icdar2015_eval/detection/iou.py:13-179), for a whole batch (csrc/db_measure.cu).

    evaluate_packed(polys, tags, offsets, boxes, count, ...)  -> dict of device tensors; never synchronises with the host, so
                                                                it can be captured in a CUDA graph, with `totals` added into
    evaluate(polygons, ignore_tags, boxes, count, ...)        -> the same, from per-image gt tensors (db_targets.pack)
    combine(totals)                                           -> combine_results' {'precision', 'recall', 'hmean'}
    QuadMeasurer().measure / validate_measure / evaluate_measure / gather_measure -> the reference's structures

gt polygons come packed as db_targets.pack and make_targets_packed give them (the validated quads and updated ignore tags);
detections as boxes_from_maps returns them.  The shapely calls of the evaluator are restated for 4-point rings
(csrc/db_measure_core.cuh): validity from GEOS's rules with exact orientation signs, the intersection by convex clipping,
the union as area(a) + area(b) - intersection (DESIGN §7).  Quads only.  CUDA only; no CPU fallback."""
import numpy as np
import torch

from . import _lib
from . import db_targets

# image_status bits
BAD_OFFSETS, BAD_COUNT = 1, 2


def _stream():
    return torch.cuda.current_stream().cuda_stream


def evaluate_packed(polys, tags, offsets, boxes, count, iou_constraint=0.5, area_precision_constraint=0.5, totals=None,
                    with_iou=False):
    """evaluate_image for the N = offsets.numel() - 1 images of a batch; no host synchronisation.

    polys [capacity, 4, 2] float32 / float64, tags uint8 [capacity], offsets int32 [N + 1] (db_targets.pack); boxes
    [N, max_dets, 4, 2] int32 / float64 and count int32 [N] (boxes_from_maps); totals, optional int64 [3] on the same device,
    is added into: care gt, care det, matched.  Returns gt_index, gt_match [capacity] (index among the image's valid gt and
    the matched det's valid index, -1 for none), det_index, det_match [N, max_dets] (likewise), det_dontcare uint8
    [N, max_dets], counts int32 [N, 5] (care gt, care det, matched, valid gt, valid det), metrics float64 [N, 3] (precision,
    recall, hmean), status int32 [N] (BAD_OFFSETS, BAD_COUNT; such an image adds nothing to totals) and, with with_iou, iou
    float64 [capacity, max_dets] (0 outside valid pairs of one image)."""
    for name, t in (("polygons", polys), ("ignore_tags", tags), ("offsets", offsets), ("boxes", boxes), ("count", count)):
        if not (torch.is_tensor(t) and t.is_cuda):
            raise NotImplementedError("megreader_b200: db_measure runs on CUDA only (no CPU fallback); %s is not a CUDA tensor" % name)
    if polys.dtype not in (torch.float32, torch.float64) or polys.dim() != 3 or polys.shape[1:] != (4, 2):
        raise RuntimeError("db_measure: gt polygons must be float32 or float64 [capacity, 4, 2], got %s %s" % (polys.dtype, tuple(polys.shape)))
    cap = polys.size(0)
    if tags.dtype != torch.uint8 or tags.shape != (cap,) or offsets.dtype != torch.int32 or offsets.dim() != 1 or offsets.numel() < 2:
        raise RuntimeError("db_measure: ignore_tags must be uint8 [capacity] and offsets int32 [N + 1]")
    N = offsets.numel() - 1
    if boxes.dtype not in (torch.int32, torch.float64) or boxes.dim() != 4 or boxes.size(0) != N or boxes.shape[2:] != (4, 2):
        raise RuntimeError("db_measure: boxes must be int32 or float64 [N, max_dets, 4, 2] with N = %d, got %s %s"
                           % (N, boxes.dtype, tuple(boxes.shape)))
    if count.dtype != torch.int32 or count.shape != (N,):
        raise RuntimeError("db_measure: count must be int32 [N] with N = %d, got %s %s" % (N, count.dtype, tuple(count.shape)))
    dev = polys.device
    for name, t in (("ignore_tags", tags), ("offsets", offsets), ("boxes", boxes), ("count", count)):
        if t.device != dev:
            raise RuntimeError("db_measure: %s is on %s, the gt polygons on %s" % (name, t.device, dev))
    if totals is not None and (not torch.is_tensor(totals) or totals.dtype != torch.int64 or totals.shape != (3,)
                               or not totals.is_contiguous() or totals.device != dev):
        raise RuntimeError("db_measure: totals must be a contiguous int64 [3] tensor on %s" % dev)
    polys, tags, offsets, boxes, count = (t.contiguous() for t in (polys, tags, offsets, boxes, count))
    maxd = boxes.size(1)
    L = _lib.lib()
    nbytes = int(L.mr_db_measure_workspace_bytes(N, cap, maxd))
    if nbytes <= 0:
        raise RuntimeError("db_measure: unsupported sizes N=%d, capacity=%d, max_dets=%d" % (N, cap, maxd))
    i32 = dict(dtype=torch.int32, device=dev)
    out = dict(gt_index=torch.empty((cap,), **i32), gt_match=torch.empty((cap,), **i32), det_index=torch.empty((N, maxd), **i32),
               det_match=torch.empty((N, maxd), **i32), det_dontcare=torch.empty((N, maxd), dtype=torch.uint8, device=dev),
               counts=torch.empty((N, 5), **i32), metrics=torch.empty((N, 3), dtype=torch.float64, device=dev),
               status=torch.empty((N,), **i32))
    if with_iou:
        out["iou"] = torch.empty((cap, maxd), dtype=torch.float64, device=dev)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.mr_db_measure(polys.data_ptr(), int(polys.dtype == torch.float64), tags.data_ptr(), offsets.data_ptr(), N, cap,
                                   boxes.data_ptr(), int(boxes.dtype == torch.float64), count.data_ptr(), maxd,
                                   float(iou_constraint), float(area_precision_constraint), ws.data_ptr(), nbytes,
                                   out["gt_index"].data_ptr(), out["gt_match"].data_ptr(), out["det_index"].data_ptr(),
                                   out["det_dontcare"].data_ptr(), out["det_match"].data_ptr(), out["counts"].data_ptr(),
                                   out["metrics"].data_ptr(), out["status"].data_ptr(),
                                   out["iou"].data_ptr() if with_iou else None,
                                   totals.data_ptr() if totals is not None else None, _stream()), "db_measure")
    out["workspace"] = ws
    return out


def evaluate(polygons, ignore_tags, boxes, count, iou_constraint=0.5, area_precision_constraint=0.5, totals=None, with_iou=False):
    """evaluate_packed for per-image gt: polygons[n] [k_n, 4, 2] float32 / float64 and ignore_tags[n] [k_n] CUDA tensors,
    packed with db_targets.pack; gt_index and gt_match come back as lists per image."""
    polys, tags, offsets = db_targets.pack(polygons, ignore_tags)
    out = evaluate_packed(polys, tags, offsets, boxes, count, iou_constraint, area_precision_constraint, totals, with_iou)
    out.pop("workspace")
    counts = [int(p.size(0)) for p in polygons]
    out["gt_index"] = list(torch.split(out["gt_index"], counts))
    out["gt_match"] = list(torch.split(out["gt_match"], counts))
    if with_iou:
        out["iou"] = list(torch.split(out["iou"], counts))
    return out


def combine(totals):
    """DetectionIoUEvaluator.combine_results from the totals (care gt, care det, matched) of evaluate_packed: one host read."""
    gt, det, matched = (int(v) for v in (totals.tolist() if torch.is_tensor(totals) else totals))
    recall = 0 if gt == 0 else float(matched) / gt
    precision = 0 if det == 0 else float(matched) / det
    hmean = 0 if recall + precision == 0 else 2 * recall * precision / (recall + precision)
    return {'precision': precision, 'recall': recall, 'hmean': hmean}


class AverageMeter:
    """concern.AverageMeter: val, avg, sum, count"""

    def __init__(self):
        self.val = 0
        self.avg = 0
        self.sum = 0
        self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count
        return self


def _quads(p, what):
    a = p.detach().cpu().numpy() if torch.is_tensor(p) else np.asarray(p)
    if a.size == 0:
        return np.zeros((0, 4, 2), a.dtype if a.dtype in (np.float32, np.float64) else np.float64)
    if a.ndim != 3 or a.shape[1:] != (4, 2):
        raise ValueError("db_measure.QuadMeasurer: %s must be quads [k, 4, 2], got shape %s (only 4-point polygons are supported)"
                         % (what, a.shape))
    return a


class QuadMeasurer:
    """The reference's QuadMeasurer on the device.  measure(batch, output) returns per image evaluate_image's dict (precision,
    recall, hmean, pairs, iouMat, gtPolPoints, detPolPoints, gtCare, detCare, gtDontCare, detDontCare, detMatched,
    evaluationLog).  batch['polygons'] / batch['ignore_tags'] hold per-image quads and tags (arrays or tensors); output[0] is
    represent()'s per-image box lists or the (boxes, scores, count) tensors of boxes_from_maps.  Where an image has no valid gt
    or no valid det, iouMat is [[0.0]] (the reference leaves that 1 x 1 matrix uninitialised, DESIGN §7).

    The constructor also takes, and ignores, the keywords the reference's config builder passes to every class it builds
    (concern/config.py: `cls(**args, cmd=cmd)` with `class` still in args), so the yaml's `measurer: class: QuadMeasurer`
    builds this class unchanged."""

    def __init__(self, iou_constraint=0.5, area_precision_constraint=0.5, device=None, **config_kwargs):
        self.iou_constraint = iou_constraint
        self.area_precision_constraint = area_precision_constraint
        self.device = device

    def _device(self, output0):
        if self.device is not None:
            return torch.device(self.device)
        if isinstance(output0, (tuple, list)) and len(output0) == 3 and torch.is_tensor(output0[0]):
            return output0[0].device
        return torch.device("cuda", torch.cuda.current_device())

    def measure(self, batch, output):
        dev = self._device(output[0])
        gts = [_quads(p, "batch['polygons']") for p in batch['polygons']]
        tags = [np.asarray(t.detach().cpu().numpy() if torch.is_tensor(t) else t, dtype=bool).reshape(-1) for t in batch['ignore_tags']]
        N = len(gts)
        if len(tags) != N or any(len(t) != len(g) for g, t in zip(gts, tags)):
            raise ValueError("db_measure.QuadMeasurer: batch['ignore_tags'] must hold one tag per gt polygon")
        gdt = gts[0].dtype if N and all(g.dtype == gts[0].dtype for g in gts) and gts[0].dtype in (np.float32, np.float64) \
            else np.float64
        polys, gtag, offsets = db_targets.pack([torch.from_numpy(np.ascontiguousarray(g, gdt)).to(dev) for g in gts],
                                               [torch.from_numpy(t).to(dev) for t in tags])
        pred = output[0]
        if isinstance(pred, (tuple, list)) and len(pred) == 3 and torch.is_tensor(pred[0]):
            boxes, count = pred[0], pred[2]
            if boxes.size(0) != N:
                raise ValueError("db_measure.QuadMeasurer: %d images of detections for %d of gt" % (boxes.size(0), N))
        else:
            dets = [_quads(np.asarray(p, dtype=np.float64) if len(p) else np.zeros((0, 4, 2)), "a detection") for p in pred]
            if len(dets) != N:
                raise ValueError("db_measure.QuadMeasurer: %d images of detections for %d of gt" % (len(dets), N))
            maxd = max([len(d) for d in dets] + [0])
            host = np.zeros((N, maxd, 4, 2), np.float64)
            for n, d in enumerate(dets):
                host[n, :len(d)] = d
            boxes = torch.from_numpy(host).to(dev)
            count = torch.tensor([len(d) for d in dets], dtype=torch.int32).to(dev)
        out = evaluate_packed(polys, gtag, offsets, boxes, count, self.iou_constraint, self.area_precision_constraint, with_iou=True)
        h = {k: v.cpu().numpy() for k, v in out.items() if k != "workspace"}
        if h["status"].any():
            raise RuntimeError("db_measure.QuadMeasurer: bad offsets or counts (status %s)" % h["status"].tolist())
        det_host = boxes.cpu().numpy().astype(np.float64)
        off = offsets.cpu().numpy()
        results = []
        for n in range(N):
            g0, g1 = off[n], off[n + 1]
            gi, gm = h["gt_index"][g0:g1], h["gt_match"][g0:g1]
            results.append(self._image(n, gts[n], tags[n], gi, gm, h, det_host, g0))
        return results

    def _image(self, n, gt, tag, gi, gm, h, det_host, g0):
        di, ddc = h["det_index"][n], h["det_dontcare"][n]
        gt_care, det_care, matched, ng, nd = (int(v) for v in h["counts"][n])
        gvalid = np.nonzero(gi >= 0)[0]
        dvalid = np.nonzero(di >= 0)[0]
        gt_dc = [int(gi[k]) for k in gvalid if tag[k]]
        det_dc = [int(di[j]) for j in dvalid if ddc[j]]
        pairs = [{'gt': int(gi[k]), 'det': int(gm[k])} for k in gvalid if gm[k] >= 0]
        log = "GT polygons: " + str(ng) + (" (" + str(len(gt_dc)) + " don't care)\n" if len(gt_dc) > 0 else "\n")
        log += "DET polygons: " + str(nd) + (" (" + str(len(det_dc)) + " don't care)\n" if len(det_dc) > 0 else "\n")
        for p in pairs:
            log += "Match GT #" + str(p['gt']) + " with Det #" + str(p['det']) + "\n"
        if nd > 100:
            iou_mat = []
        elif ng > 0 and nd > 0:
            iou_mat = h["iou"][g0 + gvalid][:, dvalid].tolist()
        else:
            iou_mat = [[0.0]]
        p, r, hm = (float(v) for v in h["metrics"][n])
        if gt_care > 0 and det_care == 0:
            p = 0                                       # the reference's int 0 in that branch
        return {
            'precision': p,
            'recall': r,
            'hmean': 0 if p + r == 0 else hm,
            'pairs': pairs,
            'iouMat': iou_mat,
            'gtPolPoints': [gt[k] for k in gvalid],
            'detPolPoints': [det_host[n, j] for j in dvalid],
            'gtCare': gt_care,
            'detCare': det_care,
            'gtDontCare': gt_dc,
            'detDontCare': det_dc,
            'detMatched': matched,
            'evaluationLog': log,
        }

    def validate_measure(self, batch, output):
        return self.measure(batch, output), [0]

    def evaluate_measure(self, batch, output):
        return self.measure(batch, output), np.linspace(0, batch['image'].shape[0]).tolist()

    def gather_measure(self, raw_metrics, logger=None):
        raw_metrics = [image_metrics for batch_metrics in raw_metrics for image_metrics in batch_metrics]
        result = combine([sum(m['gtCare'] for m in raw_metrics), sum(m['detCare'] for m in raw_metrics),
                          sum(m['detMatched'] for m in raw_metrics)])
        precision = AverageMeter()
        recall = AverageMeter()
        fmeasure = AverageMeter()
        precision.update(result['precision'], n=len(raw_metrics))
        recall.update(result['recall'], n=len(raw_metrics))
        fmeasure_score = 2 * precision.val * recall.val / (precision.val + recall.val + 1e-8)
        fmeasure.update(fmeasure_score)
        return {'precision': precision, 'recall': recall, 'fmeasure': fmeasure}
