"""ResNet trunks with the reference's surface and state-dict keys (backbones/resnet.py:39-335).

What the reference's trunk is (and what this file therefore reproduces, quirks included):
  * a *deep stem*: three 3x3 convs 3->64 (stride 2) ->64 ->128, each BN+ReLU, then 3x3/2 max-pool, so
    layer1 starts from 128 channels (resnet.py:190-201);
  * residual stages of width 64/128/256/512 with strides 1/2/2/2, returned as the tuple (x2, x3, x4, x5)
    instead of logits (resnet.py:245-256); `avgpool`, `fc` and `smooth` are constructed but never called —
    they still appear in the state dict, so they are constructed here too (resnet.py:210-213);
  * a `dcn=` dict switches conv2 of every unit in layers 2-4 to (modulated) deformable convolution fed by
    a zero-initialised `conv2_offset` 3x3 conv with 18 or 27 channels per deformable group
    (resnet.py:56-77,127-142,222-226).  `stage_with_dcn` is stored but never consulted (resnet.py:189).
    The offset conv carries no stride, and the BasicBlock deformable conv2 carries none either.
  * `dilations=` only reaches the 1x1 downsample conv (resnet.py:233), where it is a no-op.
  * weight init: conv ~ N(0, sqrt(2/(k*k*cout))), BN weight 1 / bias 0 (resnet.py:215-221).

The deformable units run on the sm_90a DCN kernels through `assets.ops.dcn` (megreader_b200.dcn); the
dense convolutions are library calls here — this trunk is a "next" row (SURVEY.md §8 A10), not the
measured hot path.
"""
import math
import os

import torch
import torch.nn as nn

try:                                      # the reference's repo-root config.py, when the host code is on sys.path
    import config
except ImportError:                       # standalone use: the reference's default (config.py:14)
    class config:                         # noqa: N801
        sync_bn = False

__all__ = ['ResNet', 'resnet18', 'resnet34', 'resnet50', 'resnet101', 'resnet152']

model_urls = {
    'resnet18': 'http://sceneparsing.csail.mit.edu/model/pretrained_resnet/resnet18-imagenet.pth',
    'resnet50': 'http://sceneparsing.csail.mit.edu/model/pretrained_resnet/resnet50-imagenet.pth',
    'resnet101': 'http://sceneparsing.csail.mit.edu/model/pretrained_resnet/resnet101-imagenet.pth',
}


def constant_init(module, constant, bias=0):
    nn.init.constant_(module.weight, constant)
    if getattr(module, 'bias', None) is not None:
        nn.init.constant_(module.bias, bias)


def bn(*args, **kwargs):
    """BatchNorm factory (resnet.py:26-30).  The reference picks apex SyncBatchNorm under `config.sync_bn`;
    apex is not part of this stack, torch's own SyncBatchNorm has the same parameters and buffers."""
    if getattr(config, 'sync_bn', False):
        return nn.SyncBatchNorm(*args, **kwargs)
    return nn.BatchNorm2d(*args, **kwargs)


def conv3x3(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, 3, stride, 1, bias=False)


class _DeformableSlot:
    """Mix-in: builds `conv2` (+ `conv2_offset`) and applies it; shared by both residual units."""

    def _build_conv2(self, planes, stride, dcn):
        self.with_dcn = dcn is not None
        self.with_modulated_dcn = bool(dcn.get('modulated', False)) if self.with_dcn else False
        if not self.with_dcn or dcn.get('fallback_on_stride', False):
            self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
            self._plain_conv2 = True
            return
        self._plain_conv2 = False
        groups = dcn.get('deformable_groups', 1)
        if self.with_modulated_dcn:
            from assets.ops.dcn import ModulatedDeformConv as op
            per_group = 27
        else:
            from assets.ops.dcn import DeformConv as op
            per_group = 18
        self.conv2_offset = nn.Conv2d(planes, groups * per_group, 3, padding=1)
        self.conv2 = op(planes, planes, kernel_size=3, padding=1, stride=stride, deformable_groups=groups, bias=False)

    def _apply_conv2(self, x):
        if not self.with_dcn:
            return self.conv2(x)
        # NB the reference takes this branch even when fallback_on_stride built a dense conv2; so do we.
        field = self.conv2_offset(x)
        if x.dtype != torch.float32:
            # bf16 trunk (megreader_b200.conv_engine): the deformable op is the reference's fp32 NCHW op (its fused forward
            # splits every operand into two bf16 halves internally), so hand it fp32 NCHW tensors
            x, field = x.float().contiguous(), field.float().contiguous()
        if self.with_modulated_dcn:
            return self.conv2(x, field[:, :18], field[:, -9:].sigmoid())
        return self.conv2(x, field)


class BasicBlock(nn.Module, _DeformableSlot):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, dcn=None):
        nn.Module.__init__(self)
        self.conv1 = conv3x3(inplanes, planes, stride)
        self.bn1 = bn(planes)
        self.relu = nn.ReLU(inplace=True)
        self._build_conv2(planes, 1, dcn)            # stride lives in conv1 (resnet.py:45,54,70)
        self.bn2 = bn(planes)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        y = self.relu(self.bn1(self.conv1(x)))
        y = self.bn2(self._apply_conv2(y))
        y = y + (x if self.downsample is None else self.downsample(x))
        return self.relu(y)


class Bottleneck(nn.Module, _DeformableSlot):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, dcn=None):
        nn.Module.__init__(self)
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = bn(planes)
        self._build_conv2(planes, stride, dcn)       # stride lives in conv2 (resnet.py:124,141)
        self.bn2 = bn(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = bn(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride
        self.dcn = dcn

    def forward(self, x):
        y = self.relu(self.bn1(self.conv1(x)))
        y = self.relu(self.bn2(self._apply_conv2(y)))
        y = self.bn3(self.conv3(y))
        y = y + (x if self.downsample is None else self.downsample(x))
        return self.relu(y)


class ResNet(nn.Module):
    STAGE_WIDTHS = (64, 128, 256, 512)

    def __init__(self, block, layers, num_classes=1000, dcn=None, stage_with_dcn=(False, False, False, False),
                 dilations=[1, 1, 1, 1]):
        super().__init__()
        self.dcn = dcn
        self.stage_with_dcn = stage_with_dcn
        self.inplanes = 128
        stem = ((3, 64, 2), (64, 64, 1), (64, 128, 1))
        for i, (cin, cout, stride) in enumerate(stem, 1):
            setattr(self, 'conv%d' % i, conv3x3(cin, cout, stride))
            setattr(self, 'bn%d' % i, bn(cout))
            setattr(self, 'relu%d' % i, nn.ReLU(inplace=True))
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        for i, width in enumerate(self.STAGE_WIDTHS):
            stage = self._make_layer(block, width, layers[i], stride=1 if i == 0 else 2,
                                     dcn=None if i == 0 else dcn, dilation=dilations[i])
            setattr(self, 'layer%d' % (i + 1), stage)
        self.avgpool = nn.AvgPool2d(7, stride=1)
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        self.smooth = nn.Conv2d(2048, 256, kernel_size=1, stride=1, padding=1)
        self._reset_parameters()

    def _reset_parameters(self):
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                fan = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2.0 / fan))
            elif isinstance(m, (nn.BatchNorm2d, nn.SyncBatchNorm)):
                m.weight.data.fill_(1)
                m.bias.data.zero_()
        if self.dcn is not None:
            for m in self.modules():
                if isinstance(m, (Bottleneck, BasicBlock)) and hasattr(m, 'conv2_offset'):
                    constant_init(m.conv2_offset, 0)

    def _make_layer(self, block, planes, blocks, stride=1, dcn=None, dilation=1):
        out_planes = planes * block.expansion
        shortcut = None
        if stride != 1 or self.inplanes != out_planes:
            shortcut = nn.Sequential(
                nn.Conv2d(self.inplanes, out_planes, 1, stride, bias=False, dilation=dilation), bn(out_planes))
        units = [block(self.inplanes, planes, stride, shortcut, dcn=dcn)]
        self.inplanes = out_planes
        units += [block(out_planes, planes, dcn=dcn) for _ in range(blocks - 1)]
        return nn.Sequential(*units)

    def stem(self, x):
        for i in (1, 2, 3):
            x = getattr(self, 'relu%d' % i)(getattr(self, 'bn%d' % i)(getattr(self, 'conv%d' % i)(x)))
        return self.maxpool(x)

    def forward(self, x):
        x2 = self.layer1(self.stem(x))
        x3 = self.layer2(x2)
        x4 = self.layer3(x3)
        x5 = self.layer4(x4)
        return x2, x3, x4, x5


def _load_pretrained(model, name):
    """`pretrained=True` in the reference downloads ImageNet weights with model_zoo (resnet.py:265-268).
    Offline boxes cannot: a local file named by MEGREADER_B200_PRETRAINED_DIR/<name>-imagenet.pth is used
    when present; otherwise this raises instead of silently training from scratch."""
    root = os.environ.get('MEGREADER_B200_PRETRAINED_DIR')
    local = os.path.join(root, name + '-imagenet.pth') if root else None
    if local and os.path.exists(local):
        state = torch.load(local, map_location='cpu')
    else:
        if name not in model_urls:
            raise KeyError(name)                 # same failure as the reference for resnet34/152
        import torch.utils.model_zoo as model_zoo
        state = model_zoo.load_url(model_urls[name])
    model.load_state_dict(state, strict=False)


_DEPTHS = {'resnet18': (BasicBlock, (2, 2, 2, 2)), 'resnet34': (BasicBlock, (3, 4, 6, 3)),
           'resnet50': (Bottleneck, (3, 4, 6, 3)), 'resnet101': (Bottleneck, (3, 4, 23, 3)),
           'resnet152': (Bottleneck, (3, 8, 36, 3))}


def _factory(name):
    block, depths = _DEPTHS[name]

    def make(pretrained=True, **kwargs):
        model = ResNet(block, list(depths), **kwargs)
        if pretrained:
            _load_pretrained(model, name)
        return model
    make.__name__ = make.__qualname__ = name
    make.__doc__ = 'ResNet trunk %s (reference backbones/resnet.py:259-335).' % name
    return make


resnet18, resnet34, resnet50, resnet101, resnet152 = (_factory(n) for n in _DEPTHS)


def deformable_resnet50(pretrained=True, **kwargs):
    """ResNet-50 with modulated DCN in layers 2-4 (resnet.py:295-309)."""
    model = ResNet(Bottleneck, [3, 4, 6, 3], dcn=dict(modulated=True, deformable_groups=1, fallback_on_stride=False),
                   stage_with_dcn=[False, True, True, True], **kwargs)
    if pretrained:
        _load_pretrained(model, 'resnet50')
    return model
