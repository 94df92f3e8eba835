"""BalanceCrossEntropyLoss of the reference (decoders/balance_cross_entropy_loss.py:5-56) as the framework composition it is,
host synchronisations and torch.topk included.  It is the comparator of the fused device loss (megreader_b200.db_head), which
computes the same value without leaving the device.

pred and gt are [N,1,H,W] and mask is [N,H,W]; like the reference, gt * mask broadcasts to [N,N,H,W], so every sample's gt is
weighed against every sample's mask (for N = 1 this is the per-pixel formula)."""
import torch
import torch.nn as nn


class BalanceCrossEntropyLoss(nn.Module):
    def __init__(self, negative_ratio=3.0, eps=1e-6):
        super().__init__()
        self.negative_ratio = negative_ratio
        self.eps = eps

    def forward(self, pred, gt, mask, return_origin=False):
        positive = (gt * mask).byte()
        negative = ((1 - gt) * mask).byte()
        n_pos = int(positive.float().sum())
        n_neg = min(int(negative.float().sum()), int(n_pos * self.negative_ratio))
        loss = nn.functional.binary_cross_entropy(pred, gt, reduction='none')[:, 0, :, :]
        pos_loss = loss * positive.float()
        neg_loss, _ = torch.topk((loss * negative.float()).view(-1), n_neg)
        balance = (pos_loss.sum() + neg_loss.sum()) / (n_pos + n_neg + self.eps)
        if return_origin:
            return balance, loss
        return balance
