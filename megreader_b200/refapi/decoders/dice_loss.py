"""DiceLoss of the reference (decoders/dice_loss.py:9-41) as the framework composition it is: 1 - 2 I / U with
I = sum(pred * gt * mask) and U = sum(pred * mask) + sum(gt * mask) + eps.  The fused L1BalanceCELoss (megreader_b200.db_head)
computes the same dice term on the device; this module is the plain composition users of `decoders.DiceLoss` expect.
InstanceDiceLoss (host-side connected components) is not provided."""
import torch.nn as nn


class DiceLoss(nn.Module):
    def __init__(self, eps=1e-6):
        super().__init__()
        self.eps = eps

    def forward(self, pred, gt, mask, weights=None):
        assert pred.dim() == 4, pred.dim()
        return self._compute(pred, gt, mask, weights)

    def _compute(self, pred, gt, mask, weights):
        if pred.dim() == 4:
            pred, gt = pred[:, 0, :, :], gt[:, 0, :, :]
        assert pred.shape == gt.shape and pred.shape == mask.shape
        if weights is not None:
            assert weights.shape == mask.shape
            mask = weights * mask
        inter = (pred * gt * mask).sum()
        union = (pred * mask).sum() + (gt * mask).sum() + self.eps
        loss = 1 - 2.0 * inter / union
        assert loss <= 1
        return loss
