"""float64 restatement of the DB detector tail and of L1BalanceCELoss (decoders/seg_detector.py, seg_detector_loss.py,
balance_cross_entropy_loss.py, dice_loss.py, l1_loss.py), the comparator of megreader_b200.db_head.  Gradients come from autograd.

It restates exactly what the reference computes: sigmoid + step function, torch's binary_cross_entropy (log clamped at -100),
the uint8 truncation of gt * mask and (1 - gt) * mask with the reference's [N,1,H,W] x [N,H,W] -> [N,N,H,W] broadcast,
k = min(#negative, int(#positive * negative_ratio)) and the sum of the k largest negative losses.  Negatives tied at the k-th
largest value tau share the remaining selection equally (weight (k - #above) / #tied each): the value is that of torch.topk,
the gradient is the deterministic rule of the CUDA implementation.  Pinned to the reference modules by tests/test_seg_detector_cpu.py."""
from collections import OrderedDict

import torch
import torch.nn.functional as F


def step(zb, zt, k):
    b = torch.sigmoid(zb.double())
    if zt is None:
        return b, None, None
    t = torch.sigmoid(zt.double())
    return b, t, torch.reciprocal(1 + torch.exp(-k * (b - t)))


def balance_weights(gt, mask):
    """(positive, negative) [N,N,H,W] float64 from the fp32 products the reference truncates."""
    g, m = gt.detach().float(), mask.detach().float()
    return (g * m).trunc().double(), ((1 - g) * m).trunc().double()


def topk_sum(v, k):
    """sum of the k largest entries of the flat float64 tensor v, ties at tau weighted (k - #above) / #tied."""
    if k == 0:
        return v.sum() * 0
    vd = v.detach()
    tau = torch.topk(vd, k).values[-1]
    above, tied = vd > tau, vd == tau
    w = above.double() + tied.double() * (k - int(above.sum())) / int(tied.sum())
    return (v * w).sum()


def balance_bce(binary, gt, mask, negative_ratio=3.0, eps=1e-6):
    positive, negative = balance_weights(gt, mask)
    n_pos = int(positive.sum())
    k = min(int(negative.sum()), int(n_pos * negative_ratio))
    loss = F.binary_cross_entropy(binary.double(), gt.double(), reduction='none')[:, 0]
    pos = (loss * positive).sum()
    return (pos + topk_sum((loss * negative).reshape(-1), k)) / (n_pos + k + eps)


def dice(pred, gt, mask, eps=1e-6):
    p, g, m = pred.double()[:, 0], gt.double()[:, 0], mask.double()
    inter = (p * g * m).sum()
    union = (p * m).sum() + (g * m).sum() + eps
    return 1 - 2.0 * inter / union


def mask_l1(pred, gt, mask):
    m = mask.double()
    return (torch.abs(pred.double()[:, 0] - gt.double()) * m).sum() / m.sum()


def l1_balance_ce(pred, batch, eps=1e-6, l1_scale=10, bce_scale=5, negative_ratio=3.0, bce_eps=1e-6):
    """-> (loss, {bce_loss, thresh_loss, l1_loss}), float64."""
    bce = balance_bce(pred['binary'], batch['gt'], batch['mask'], negative_ratio, bce_eps)
    l1 = mask_l1(pred['thresh'], batch['thresh_map'], batch['thresh_mask'])
    d = dice(pred['thresh_binary'], batch['gt'], batch['mask'], eps)
    return d + l1_scale * l1 + bce * bce_scale, dict(bce_loss=bce, thresh_loss=d, l1_loss=l1)


def seg_detector_forward(head, features):
    """The forward of a (refapi or reference) SegDetector module with this file's float64 tail: the module's own
    convolutions / BatchNorms / upsampling in the dtype of its parameters, binarize[:-1] / thresh[:-1], then step()."""
    c2, c3, c4, c5 = features
    in5, in4, in3, in2 = head.in5(c5), head.in4(c4), head.in3(c3), head.in2(c2)
    out4 = head.up5(in5) + in4
    out3 = head.up4(out4) + in3
    out2 = head.up3(out3) + in2
    fuse = torch.cat((head.out5(in5), head.out4(out4), head.out3(out3), head.out2(out2)), 1)
    zb = head.binarize[:-1](fuse)
    if not head.adaptive:
        return OrderedDict(binary=step(zb, None, head.k)[0])
    if head.serial:
        fuse = torch.cat((fuse, F.interpolate(step(zb, None, head.k)[0].to(fuse.dtype), fuse.shape[2:])), 1)
    b, t, s = step(zb, head.thresh[:-1](fuse), head.k)
    return OrderedDict(binary=b, thresh=t, thresh_binary=s)
