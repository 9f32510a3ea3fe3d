"""Temporal models with spatial layers between the temporal blocks (MODEL.TEMPORAL_MODEL.INBETWEEN_LAYERS > 0), built from the oracle's
modules: ``Bottleneck3D`` restates fiery/layers/temporal.py:120-164 with the reference's attribute names, and
``temporal_model(..., inbetween_layers=n)`` inserts n of them after each block as fiery/models/temporal_model.py:20-41 does, so the
``state_dict`` keys are the reference's."""
from collections import OrderedDict

import torch.nn as nn

from oracle import temporal_oracle as TO


class Bottleneck3D(nn.Module):
    """1x1x1 down-projection, a causal (1, 3, 3) convolution, 1x1x1 up-projection, plus a skip (a 1x1x1 conv + bn when the channel
    count changes)."""

    def __init__(self, in_channels, out_channels=None, kernel_size=(2, 3, 3)):
        super().__init__()
        mid = in_channels // 2
        out_channels = out_channels or in_channels
        self.layers = nn.Sequential(OrderedDict([
            ("conv_down_project", TO.conv_1x1x1_norm_activated(in_channels, mid)),
            ("conv", TO.CausalConv3d(mid, mid, kernel_size=kernel_size)),
            ("conv_up_project", TO.conv_1x1x1_norm_activated(mid, out_channels)),
        ]))
        self.projection = None if out_channels == in_channels else nn.Sequential(
            nn.Conv3d(in_channels, out_channels, kernel_size=1, bias=False), nn.BatchNorm3d(out_channels))

    def forward(self, x):
        return self.layers(x) + (self.projection(x) if self.projection is not None else x)


def temporal_model(in_channels, receptive_field, input_shape, start_out_channels=64, inbetween_layers=0, **kw):
    m = TO.TemporalModel(in_channels, receptive_field, input_shape, start_out_channels=start_out_channels, **kw)
    if inbetween_layers:
        mods = []
        for blk in m.model:
            mods.append(blk)
            mods.extend(Bottleneck3D(blk.out_channels, blk.out_channels, kernel_size=(1, 3, 3)) for _ in range(inbetween_layers))
        m.model = nn.Sequential(*mods)
    return m
