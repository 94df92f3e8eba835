"""MaskL1Loss of the reference (decoders/l1_loss.py:5-11): sum(|pred[:, 0] - gt| * mask) / sum(mask), returned with the metric
dict {'l1_loss': loss}.  A plain framework composition; the fused L1BalanceCELoss computes the same term on the device."""
import torch
import torch.nn as nn


class MaskL1Loss(nn.Module):
    def forward(self, pred, gt, mask):
        loss = (torch.abs(pred[:, 0] - gt) * mask).sum() / mask.sum()
        return loss, dict(l1_loss=loss)
