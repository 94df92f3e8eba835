"""DB text detector head with the reference's surface (decoders/seg_detector.py): constructor, submodule layout and state-dict
keys in2..in5, out2..out5, binarize.{0,1,3,4,6}.*, thresh.{0,1,3,4,6}.*.

The convolutions, BatchNorms and 2x2 transposed convolutions are ordinary nn modules, so megreader_b200.conv_engine can put them
on the wgmma kernels.  Forward runs binarize[:-1] / thresh[:-1] (everything but the final nn.Sigmoid, which stays in the Sequential
for key parity) and hands both logit maps to one fused node, megreader_b200.db_head.StepFunction: the two sigmoids and the step
function 1 / (1 + exp(-k (binary - thresh))) in one CUDA pass each way."""
from collections import OrderedDict

import torch
import torch.nn as nn

from megreader_b200.db_head import step_function


class SegDetector(nn.Module):
    def __init__(self, in_channels=[64, 128, 256, 512], inner_channels=256, k=10, bias=False, adaptive=False, smooth=False,
                 serial=False, *args, **kwargs):
        super().__init__()
        self.k = k
        self.serial = serial
        self.up5 = nn.Upsample(scale_factor=2, mode='nearest')
        self.up4 = nn.Upsample(scale_factor=2, mode='nearest')
        self.up3 = nn.Upsample(scale_factor=2, mode='nearest')
        q = inner_channels // 4
        self.in5 = nn.Conv2d(in_channels[-1], inner_channels, 1, bias=bias)
        self.in4 = nn.Conv2d(in_channels[-2], inner_channels, 1, bias=bias)
        self.in3 = nn.Conv2d(in_channels[-3], inner_channels, 1, bias=bias)
        self.in2 = nn.Conv2d(in_channels[-4], inner_channels, 1, bias=bias)
        self.out5 = nn.Sequential(nn.Conv2d(inner_channels, q, 3, padding=1, bias=bias), nn.Upsample(scale_factor=8, mode='nearest'))
        self.out4 = nn.Sequential(nn.Conv2d(inner_channels, q, 3, padding=1, bias=bias), nn.Upsample(scale_factor=4, mode='nearest'))
        self.out3 = nn.Sequential(nn.Conv2d(inner_channels, q, 3, padding=1, bias=bias), nn.Upsample(scale_factor=2, mode='nearest'))
        self.out2 = nn.Conv2d(inner_channels, q, 3, padding=1, bias=bias)
        self.binarize = nn.Sequential(
            nn.Conv2d(inner_channels, q, 3, padding=1, bias=bias), nn.BatchNorm2d(q), nn.ReLU(inplace=True),
            nn.ConvTranspose2d(q, q, 2, 2), nn.BatchNorm2d(q), nn.ReLU(inplace=True),
            nn.ConvTranspose2d(q, 1, 2, 2), nn.Sigmoid())
        self.binarize.apply(self.weights_init)
        self.adaptive = adaptive
        if adaptive:
            self.thresh = self._init_thresh(inner_channels, serial=serial, smooth=smooth, bias=bias)
            self.thresh.apply(self.weights_init)
        for m in (self.in5, self.in4, self.in3, self.in2, self.out5, self.out4, self.out3, self.out2):
            m.apply(self.weights_init)

    def weights_init(self, m):
        name = m.__class__.__name__
        if 'Conv' in name:
            nn.init.kaiming_normal_(m.weight.data)
        elif 'BatchNorm' in name:
            m.weight.data.fill_(1.)
            m.bias.data.fill_(1e-4)

    def _init_thresh(self, inner_channels, serial=False, smooth=False, bias=False):
        q = inner_channels // 4
        self.thresh = nn.Sequential(
            nn.Conv2d(inner_channels + (1 if serial else 0), q, 3, padding=1, bias=bias), nn.BatchNorm2d(q), nn.ReLU(inplace=True),
            self._init_upsample(q, q, smooth=smooth, bias=bias), nn.BatchNorm2d(q), nn.ReLU(inplace=True),
            self._init_upsample(q, 1, smooth=smooth, bias=bias), nn.Sigmoid())
        return self.thresh

    def _init_upsample(self, in_channels, out_channels, smooth=False, bias=False):
        if not smooth:
            return nn.ConvTranspose2d(in_channels, out_channels, 2, 2)
        inter = in_channels if out_channels == 1 else out_channels
        layers = [nn.Upsample(scale_factor=2, mode='nearest'), nn.Conv2d(in_channels, inter, 3, 1, 1, bias=bias)]
        if out_channels == 1:
            layers.append(nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=1, bias=True))
        # as in the reference: nn.Sequential is handed the list itself, which it refuses, so smooth=True fails here
        return nn.Sequential(layers)

    def forward(self, features, gt=None, masks=None, training=False):
        c2, c3, c4, c5 = features
        in5, in4, in3, in2 = self.in5(c5), self.in4(c4), self.in3(c3), self.in2(c2)
        out4 = self.up5(in5) + in4
        out3 = self.up4(out4) + in3
        out2 = self.up3(out3) + in2
        fuse = torch.cat((self.out5(in5), self.out4(out4), self.out3(out3), self.out2(out2)), 1)
        zb = self.binarize[:-1](fuse)
        if not self.adaptive:
            binary, _, _ = step_function(zb, None, self.k)
            return OrderedDict(binary=binary)
        if self.serial:
            binary, _, _ = step_function(zb, None, self.k)
            fuse = torch.cat((fuse, nn.functional.interpolate(binary, fuse.shape[2:])), 1)
        zt = self.thresh[:-1](fuse)
        binary, thresh, thresh_binary = step_function(zb, zt.to(zb.dtype), self.k)
        return OrderedDict(binary=binary, thresh=thresh, thresh_binary=thresh_binary)

    def step_function(self, x, y):
        return torch.reciprocal(1 + torch.exp(-self.k * (x - y)))
