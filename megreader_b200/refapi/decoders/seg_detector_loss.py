"""Criteria of the DB detector with the reference's surface (decoders/seg_detector_loss.py).  Every criterion takes
(pred, batch) with pred = SegDetector's dict (binary, thresh, thresh_binary) and batch = the DB batch (gt [N,1,H,W]; mask,
thresh_map, thresh_mask [N,H,W]) and returns (loss, metrics).

L1BalanceCELoss, the criterion of seg_detector_db.yaml, is one fused autograd node on csrc/db_head.cu
(megreader_b200.db_head.L1BalanceCELossFunction): hard-negative mining without host synchronisation, so the training step can
be captured in a CUDA graph.  DiceLoss / AdaptiveDiceLoss / L1DiceLoss are short framework compositions of decoders.DiceLoss
and decoders.MaskL1Loss.  The instance-dice and leaky-dice criteria are not provided."""
import sys

import torch.nn as nn

from megreader_b200.db_head import l1_balance_ce_loss


class SegDetectorLossBuilder():
    """SegDetectorLossBuilder(name, *args, **kwargs).build() -> the criterion class of that name in this module."""

    def __init__(self, loss_class, *args, **kwargs):
        self.loss_class = loss_class
        self.loss_args = args
        self.loss_kwargs = kwargs

    def build(self):
        return getattr(sys.modules[__name__], self.loss_class)(*self.loss_args, **self.loss_kwargs)


class DiceLoss(nn.Module):
    """Dice on `binary` (SegDetector without the adaptive branch)."""

    def __init__(self, eps=1e-6):
        super().__init__()
        from .dice_loss import DiceLoss as Dice
        self.loss = Dice(eps)

    def forward(self, pred, batch):
        loss = self.loss(pred['binary'], batch['gt'], batch['mask'])
        return loss, dict(dice_loss=loss)


class AdaptiveDiceLoss(nn.Module):
    """Dice on `binary` plus dice on `thresh_binary`."""

    def __init__(self, eps=1e-6):
        super().__init__()
        from .dice_loss import DiceLoss as Dice
        self.main_loss = Dice(eps)
        self.thresh_loss = Dice(eps)

    def forward(self, pred, batch):
        main = self.main_loss(pred['binary'], batch['gt'], batch['mask'])
        thresh = self.thresh_loss(pred['thresh_binary'], batch['gt'], batch['mask'])
        return main + thresh, dict(main_loss=main, thresh_loss=thresh)


class L1DiceLoss(nn.Module):
    """AdaptiveDiceLoss plus l1_scale * MaskL1Loss on `thresh`."""

    def __init__(self, eps=1e-6, l1_scale=10):
        super().__init__()
        from .l1_loss import MaskL1Loss
        self.dice_loss = AdaptiveDiceLoss(eps=eps)
        self.l1_loss = MaskL1Loss()
        self.l1_scale = l1_scale

    def forward(self, pred, batch):
        dice, metrics = self.dice_loss(pred, batch)
        l1, l1_metric = self.l1_loss(pred['thresh'], batch['thresh_map'], batch['thresh_mask'])
        metrics.update(**l1_metric)
        return dice + self.l1_scale * l1, metrics


class L1BalanceCELoss(nn.Module):
    """bce_scale * BalanceCrossEntropyLoss(binary) + l1_scale * MaskL1Loss(thresh) + DiceLoss(thresh_binary), fused.
    metrics = {bce_loss, thresh_loss (the dice term), l1_loss}.  The dice term's `assert loss <= 1` of the reference is not
    evaluated: it would need a host synchronisation."""

    def __init__(self, eps=1e-6, l1_scale=10, bce_scale=5):
        super().__init__()
        from .dice_loss import DiceLoss as Dice
        from .l1_loss import MaskL1Loss
        from .balance_cross_entropy_loss import BalanceCrossEntropyLoss
        self.dice_loss = Dice(eps=eps)
        self.l1_loss = MaskL1Loss()
        self.bce_loss = BalanceCrossEntropyLoss()
        self.l1_scale = l1_scale
        self.bce_scale = bce_scale

    def forward(self, pred, batch):
        loss, bce, dice, l1 = l1_balance_ce_loss(
            pred['binary'], pred['thresh'], pred['thresh_binary'], batch['gt'], batch['mask'], batch['thresh_map'],
            batch['thresh_mask'], eps=self.dice_loss.eps, l1_scale=self.l1_scale, bce_scale=self.bce_scale,
            negative_ratio=self.bce_loss.negative_ratio, bce_eps=self.bce_loss.eps)
        return loss, dict(bce_loss=bce, thresh_loss=dice, l1_loss=l1)
