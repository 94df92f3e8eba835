"""EAST detection head with the reference's surface (decoders/east.py:7-60): 3x3 conv + BN + ReLU, two 2x2 stride-2 transposed
convolutions (x4 up-sampling), a 1-channel heat-map and an 8-channel dense-box 1x1 prediction, BCE-with-logits / MSE losses
weighted per pixel and averaged per sample.  State-dict keys: head_layer.{0,1,3,4,6}.*, heatmap_pred_layer.0.*,
densebox_pred_layer.0.*.  The stride-1 convolutions are ordinary nn.Conv2d modules, i.e. megreader_b200.conv_engine can put them on
the wgmma kernels; the transposed convolutions and the element-wise losses are library (ATen) calls."""
import torch
import torch.nn as nn
import torch.nn.functional as F


class EASTDecoder(nn.Module):
    def __init__(self, channels=256, heatmap_ratio=1.0, densebox_ratio=0.01, densebox_rescale_factor=512):
        super().__init__()
        self.heatmap_ratio = heatmap_ratio
        self.densebox_ratio = densebox_ratio
        self.densebox_rescale_factor = densebox_rescale_factor
        up1, up2 = channels // 2, channels // 4
        self.head_layer = nn.Sequential(
            nn.Conv2d(channels, channels, kernel_size=3, stride=1, padding=1), nn.BatchNorm2d(channels), nn.ReLU(inplace=True),
            nn.ConvTranspose2d(channels, up1, kernel_size=2, stride=2, padding=0), nn.BatchNorm2d(up1), nn.ReLU(inplace=True),
            nn.ConvTranspose2d(up1, up2, kernel_size=2, stride=2, padding=0))
        self.heatmap_pred_layer = nn.Sequential(nn.Conv2d(up2, 1, kernel_size=1, stride=1, padding=0))
        self.densebox_pred_layer = nn.Sequential(nn.Conv2d(up2, 8, kernel_size=1, stride=1, padding=0))

    def forward(self, input, label, meta, train):
        feature = self.head_layer(input).float()
        heatmap_pred = self.heatmap_pred_layer(feature).float()
        densebox_pred = self.densebox_pred_layer(feature).float() * self.densebox_rescale_factor
        pred = {'heatmap': torch.sigmoid(heatmap_pred), 'densebox': densebox_pred}
        if not train:
            return pred
        hm_loss = F.binary_cross_entropy_with_logits(heatmap_pred, label['heatmap'], reduction='none')
        hm_loss = (hm_loss * label['heatmap_weight']).mean(dim=(1, 2, 3))
        db_loss = F.mse_loss(densebox_pred, label['densebox'], reduction='none')
        db_loss = (db_loss * label['densebox_weight']).mean(dim=(1, 2, 3))
        loss = hm_loss * self.heatmap_ratio + db_loss * self.densebox_ratio
        return loss, pred, {'heatmap_loss': hm_loss, 'densebox_loss': db_loss}
