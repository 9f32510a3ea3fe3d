"""CPU/GPU oracle for the decoder (fiery/models/decoder.py, fiery/layers/convolutions.py:203-214).  TEST INFRASTRUCTURE ONLY.

A plain-torch restatement of ``UpsamplingAdd`` and ``Decoder`` with the reference's attribute names, so ``state_dict`` keys match and a
state dict moves between the two.  The trunk is torchvision's ``resnet18(weights=None, zero_init_residual=True)`` (no download), as
the reference's ``resnet18(pretrained=False, zero_init_residual=True)`` (decoder.py:10).  Tests build their models from here;
oracle/gen_golden_decoder.py pins it against the real class.
"""
from __future__ import annotations

import torch.nn as nn
from torchvision.models.resnet import resnet18


class UpsamplingAdd(nn.Module):
    """fiery/layers/convolutions.py:203-214: bilinear x2 upsample, bias-free 1x1, BatchNorm2d, plus the skip."""

    def __init__(self, in_channels, out_channels, scale_factor=2):
        super().__init__()
        self.upsample_layer = nn.Sequential(
            nn.Upsample(scale_factor=scale_factor, mode="bilinear", align_corners=False),
            nn.Conv2d(in_channels, out_channels, kernel_size=1, padding=0, bias=False),
            nn.BatchNorm2d(out_channels),
        )

    def forward(self, x, x_skip):
        return self.upsample_layer(x) + x_skip


def output_head(channels: int, n_out: int, sigmoid: bool = False) -> nn.Sequential:
    """decoder.py:24-50: 3x3 conv (bias-free, padding 1), BatchNorm2d, ReLU(inplace), 1x1 conv with a bias[, Sigmoid]"""
    layers = [nn.Conv2d(channels, channels, kernel_size=3, padding=1, bias=False), nn.BatchNorm2d(channels), nn.ReLU(inplace=True),
              nn.Conv2d(channels, n_out, kernel_size=1, padding=0)]
    return nn.Sequential(*layers, nn.Sigmoid()) if sigmoid else nn.Sequential(*layers)


class Decoder(nn.Module):
    """decoder.py:7-91."""

    def __init__(self, in_channels, n_classes, predict_future_flow):
        super().__init__()
        backbone = resnet18(weights=None, zero_init_residual=True)
        self.first_conv = nn.Conv2d(in_channels, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = backbone.bn1
        self.relu = backbone.relu
        self.layer1 = backbone.layer1
        self.layer2 = backbone.layer2
        self.layer3 = backbone.layer3
        self.predict_future_flow = predict_future_flow
        shared_out_channels = in_channels
        self.up3_skip = UpsamplingAdd(256, 128, scale_factor=2)
        self.up2_skip = UpsamplingAdd(128, 64, scale_factor=2)
        self.up1_skip = UpsamplingAdd(64, shared_out_channels, scale_factor=2)
        self.segmentation_head = output_head(shared_out_channels, n_classes)
        self.instance_offset_head = output_head(shared_out_channels, 2)
        self.instance_center_head = output_head(shared_out_channels, 1, sigmoid=True)
        if self.predict_future_flow:
            self.instance_future_head = output_head(shared_out_channels, 2)

    def forward(self, x):
        b, s, c, h, w = x.shape
        x = x.view(b * s, c, h, w)
        skip_x = {"1": x}
        x = self.relu(self.bn1(self.first_conv(x)))
        x = self.layer1(x)
        skip_x["2"] = x
        x = self.layer2(x)
        skip_x["3"] = x
        x = self.layer3(x)
        x = self.up3_skip(x, skip_x["3"])
        x = self.up2_skip(x, skip_x["2"])
        x = self.up1_skip(x, skip_x["1"])
        seg = self.segmentation_head(x)
        center = self.instance_center_head(x)
        offset = self.instance_offset_head(x)
        flow = self.instance_future_head(x) if self.predict_future_flow else None
        return {
            "segmentation": seg.view(b, s, *seg.shape[1:]),
            "instance_center": center.view(b, s, *center.shape[1:]),
            "instance_offset": offset.view(b, s, *offset.shape[1:]),
            "instance_flow": flow.view(b, s, *flow.shape[1:]) if flow is not None else None,
        }
