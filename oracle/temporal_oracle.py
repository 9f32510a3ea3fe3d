"""CPU/GPU oracle for the temporal model (fiery/layers/temporal.py, fiery/models/temporal_model.py).  TEST INFRASTRUCTURE ONLY.

A plain-torch restatement of ``conv_1x1x1_norm_activated``, ``CausalConv3d``, ``PyramidSpatioTemporalPooling``, ``TemporalBlock``
and ``TemporalModel`` with the reference's attribute names, so ``state_dict`` keys match and a state dict moves between the two.
Tests on a machine without the reference build their models from here; oracle/gen_golden_temporal.py pins it against the real
classes (identical keys, bit-equal outputs in train and eval) and records tests/golden/temporal.npz.
"""
from __future__ import annotations

from collections import OrderedDict

import torch
import torch.nn as nn
import torch.nn.functional as F


def conv_1x1x1_norm_activated(in_channels: int, out_channels: int) -> nn.Sequential:
    """Conv3d 1x1x1 (no bias) -> BatchNorm3d -> ReLU(inplace); keys conv / norm / activation."""
    return nn.Sequential(OrderedDict([
        ("conv", nn.Conv3d(in_channels, out_channels, kernel_size=1, bias=False)),
        ("norm", nn.BatchNorm3d(out_channels)),
        ("activation", nn.ReLU(inplace=True)),
    ]))


class CausalConv3d(nn.Module):
    """Zero pad (time on the left only, space symmetric), Conv3d without padding, BatchNorm3d, ReLU."""

    def __init__(self, in_channels, out_channels, kernel_size=(2, 3, 3), dilation=(1, 1, 1), bias=False):
        super().__init__()
        kt, kh, kw = kernel_size
        pt, ph, pw = (kt - 1) * dilation[0], ((kh - 1) * dilation[1]) // 2, ((kw - 1) * dilation[2]) // 2
        self.pad = nn.ConstantPad3d(padding=(pw, pw, ph, ph, pt, 0), value=0)
        self.conv = nn.Conv3d(in_channels, out_channels, kernel_size, dilation=dilation, stride=1, padding=0, bias=bias)
        self.norm = nn.BatchNorm3d(out_channels)
        self.activation = nn.ReLU(inplace=True)

    def forward(self, x):
        return self.activation(self.norm(self.conv(self.pad(x))))


class PyramidSpatioTemporalPooling(nn.Module):
    """Per pool size (2, ph, pw): average pool (stride (1, ph, pw), one frame of zero padding in front that is not counted), 1x1x1
    conv / bn / relu, the padded last frame dropped, bilinear upsampling back to the map."""

    def __init__(self, in_channels, reduction_channels, pool_sizes):
        super().__init__()
        feats = []
        for size in pool_sizes:
            assert size[0] == 2
            feats.append(nn.Sequential(OrderedDict([
                ("avgpool", nn.AvgPool3d(kernel_size=size, stride=(1, *size[1:]), padding=(1, 0, 0), count_include_pad=False)),
                ("conv_bn_relu", conv_1x1x1_norm_activated(in_channels, reduction_channels)),
            ])))
        self.features = nn.ModuleList(feats)

    def forward(self, x):
        b, _, t, h, w = x.shape
        out = []
        for f in self.features:
            y = f(x)[:, :, :-1].contiguous()
            c = y.shape[1]
            y = F.interpolate(y.view(b * t, c, *y.shape[-2:]), (h, w), mode="bilinear", align_corners=False)
            out.append(y.view(b, c, t, h, w))
        return torch.cat(out, 1)


class TemporalBlock(nn.Module):
    """Three paths (1x1x1 -> causal (2,3,3); 1x1x1 -> causal (1,3,3); 1x1x1), optional pyramid pooling, a 1x1x1 aggregation and a
    skip that goes through a 1x1x1 conv + bn when the channel count changes."""

    def __init__(self, in_channels, out_channels=None, use_pyramid_pooling=False, pool_sizes=None):
        super().__init__()
        self.in_channels = in_channels
        self.half_channels = in_channels // 2
        self.out_channels = out_channels or in_channels
        self.kernels = [(2, 3, 3), (1, 3, 3)]
        self.use_pyramid_pooling = use_pyramid_pooling
        paths = [nn.Sequential(conv_1x1x1_norm_activated(in_channels, self.half_channels),
                               CausalConv3d(self.half_channels, self.half_channels, kernel_size=k)) for k in self.kernels]
        paths.append(conv_1x1x1_norm_activated(in_channels, self.half_channels))
        self.convolution_paths = nn.ModuleList(paths)
        agg_in = len(paths) * self.half_channels
        if use_pyramid_pooling:
            reduction = in_channels // 3
            self.pyramid_pooling = PyramidSpatioTemporalPooling(in_channels, reduction, pool_sizes)
            agg_in += len(pool_sizes) * reduction
        self.aggregation = nn.Sequential(conv_1x1x1_norm_activated(agg_in, self.out_channels))
        if self.out_channels != in_channels:
            self.projection = nn.Sequential(nn.Conv3d(in_channels, self.out_channels, kernel_size=1, bias=False),
                                            nn.BatchNorm3d(self.out_channels))
        else:
            self.projection = None

    def forward(self, x):
        res = torch.cat([p(x) for p in self.convolution_paths], dim=1)
        if self.use_pyramid_pooling:
            res = torch.cat([res, self.pyramid_pooling(x)], dim=1)
        res = self.aggregation(res)
        if self.out_channels != self.in_channels:
            x = self.projection(x)
        return x + res


class TemporalModel(nn.Module):
    """receptive_field - 1 TemporalBlocks over (b, C, s, X, Y); input and output (b, s, C, X, Y), the output from the last frame on.
    (No spatial Bottleneck3D layers: every shipped config has N_SPATIAL_LAYERS_BETWEEN_TEMPORAL_LAYERS = 0.)"""

    def __init__(self, in_channels, receptive_field, input_shape, start_out_channels=64, extra_in_channels=0,
                 use_pyramid_pooling=True):
        super().__init__()
        self.receptive_field = receptive_field
        h, w = input_shape
        blocks, cin, cout = [], in_channels, start_out_channels
        for _ in range(receptive_field - 1):
            blocks.append(TemporalBlock(cin, cout, use_pyramid_pooling=use_pyramid_pooling,
                                        pool_sizes=[(2, h, w)] if use_pyramid_pooling else None))
            cin, cout = cout, cout + extra_in_channels
        self.out_channels = cin
        self.model = nn.Sequential(*blocks)

    def forward(self, x):
        x = self.model(x.permute(0, 2, 1, 3, 4))
        return x.permute(0, 2, 1, 3, 4).contiguous()[:, (self.receptive_field - 1):]


def egopose_concat(bev: torch.Tensor, future_egomotion: torch.Tensor) -> torch.Tensor:
    """fiery.py:148-155: the egopose broadcast over the map and concatenated to the BEV, zeros at t = 0 and
    future_egomotion[:, t - 1] after that.  bev (b, s, C, X, Y), future_egomotion (b, s, E)."""
    b, s, c = future_egomotion.shape
    h, w = bev.shape[-2:]
    sp = future_egomotion.view(b, s, c, 1, 1).expand(b, s, c, h, w)
    sp = torch.cat([torch.zeros_like(sp[:, :1]), sp[:, :(s - 1)]], dim=1)
    return torch.cat([bev, sp], dim=-3)


def normwise_error(got: torch.Tensor, ref: torch.Tensor) -> float:
    ref = ref.detach().double()
    return float((got.detach().double() - ref).norm() / ref.norm().clamp_min(1e-30))
