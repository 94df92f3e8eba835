"""1-D CTC head over a conv encoder, the reference's `CTCDecoder` surface (decoders/ctc_decoder.py:14-70).

encode = the same 7-conv / 3-pool stack as the attention head; pred_conv = 1x1 conv to len(charset).
train: log_softmax over classes, first feature row, (W,N,C) -> CTC with `input_lengths = 32` for every sample,
mean reduction ( mean_b nll_b / max(len_b,1) ), no zero_infinity; returns (loss, log_probs as (N,C,W)).
eval: softmax over classes, (N,C,H,W).
The loss runs on the sm_90a 1-D CTC kernels (megreader_b200.ctc1d) fused with the log-softmax."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from megreader_b200 import ctc1d
from megreader_b200.charset import default_charset


class CTCDecoder(nn.Module):
    def __init__(self, in_channels, charset=None, inner_channels=256, **kwargs):
        super().__init__()
        charset = charset if charset is not None else default_charset()
        self.inner_channels = inner_channels
        self.encode = self._init_encoder(in_channels)
        self.pred_conv = nn.Conv2d(inner_channels, len(charset), kernel_size=1, bias=True, padding=0)
        self.softmax = nn.LogSoftmax(dim=1)
        self.blank = kwargs.get('blank', 0)

    def conv_bn_relu(self, input_channels, output_channels, kernel_size=3, stride=1, padding=1):
        return nn.Sequential(nn.Conv2d(input_channels, output_channels, kernel_size, stride, padding),
                             nn.BatchNorm2d(output_channels), nn.ReLU(inplace=True))

    def _init_encoder(self, in_channels, stride=(2, 1), padding=(0, 1)):
        c = self.inner_channels
        cbr = self.conv_bn_relu
        return nn.Sequential(cbr(in_channels, c), cbr(c, c), nn.MaxPool2d((2, 2), (2, 2), (0, 0)),
                             cbr(c, c), cbr(c, c), nn.MaxPool2d(stride, stride, (0, 0)),
                             cbr(c, c), cbr(c, c), nn.MaxPool2d(stride, stride, (0, 0)),
                             cbr(c, c, kernel_size=(2, 3), stride=stride, padding=padding))

    def forward(self, feature, targets=None, lengths=None, train=False):
        pred = self.pred_conv(self.encode(feature))
        if not train:
            return F.softmax(pred, dim=1)
        logits = pred.select(2, 0).permute(2, 0, 1).contiguous()                  # (W,N,C)
        n = feature.size(0)
        input_lengths = torch.full((n,), 32, dtype=torch.int32)                   # ctc_decoder.py:63 hard-codes 32
        loss, log_probs = ctc1d.ctc_loss_from_logits(logits, targets, input_lengths, lengths, blank=0,
                                                     reduction='mean', zero_infinity=False)
        return loss, log_probs.permute(1, 2, 0)
