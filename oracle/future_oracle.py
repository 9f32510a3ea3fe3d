"""CPU/GPU oracle for the future prediction (fiery/layers/temporal.py:10-62, fiery/layers/convolutions.py, fiery/models/
future_prediction.py).  TEST INFRASTRUCTURE ONLY.

A plain-torch restatement of ``ConvBlock`` (3x3, BatchNorm2d, ReLU), ``Bottleneck`` (the plain variant FuturePrediction builds),
``SpatialGRU`` (without flow warping) and ``FuturePrediction`` with the reference's attribute names, so ``state_dict`` keys match and a
state dict moves between the two.  Tests build their models from here; oracle/gen_golden_future.py pins it against the real classes.
"""
from __future__ import annotations

from collections import OrderedDict

import torch
import torch.nn as nn


class ConvBlock(nn.Module):
    """Conv2d (kernel k, padding (k - 1) / 2, stride 1) -> BatchNorm2d -> ReLU(inplace); keys conv / norm / activation."""

    def __init__(self, in_channels, out_channels=None, kernel_size=3, bias=False):
        super().__init__()
        out_channels = out_channels or in_channels
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, 1, padding=(kernel_size - 1) // 2, bias=bias)
        self.norm = nn.BatchNorm2d(out_channels)
        self.activation = nn.ReLU(inplace=True)

    def forward(self, x):
        return self.activation(self.norm(self.conv(x)))


class Bottleneck(nn.Module):
    """1x1 down projection, 3x3 conv, 1x1 up projection, each with BatchNorm2d + ReLU, dropout p = 0, plus the input."""

    def __init__(self, in_channels, kernel_size=3):
        super().__init__()
        mid = in_channels // 2
        self.layers = nn.Sequential(OrderedDict([
            ("conv_down_project", nn.Conv2d(in_channels, mid, kernel_size=1, bias=False)),
            ("abn_down_project", nn.Sequential(nn.BatchNorm2d(mid), nn.ReLU(inplace=True))),
            ("conv", nn.Conv2d(mid, mid, kernel_size=kernel_size, bias=False, dilation=1, padding=(kernel_size - 1) // 2, groups=1)),
            ("abn", nn.Sequential(nn.BatchNorm2d(mid), nn.ReLU(inplace=True))),
            ("conv_up_project", nn.Conv2d(mid, in_channels, kernel_size=1, bias=False)),
            ("abn_up_project", nn.Sequential(nn.BatchNorm2d(in_channels), nn.ReLU(inplace=True))),
            ("dropout", nn.Dropout2d(p=0.0)),
        ]))
        self.projection = None

    def forward(self, *args):
        (x,) = args
        return self.layers(x) + x


class SpatialGRU(nn.Module):
    """The reference's convolutional GRU over (b, T, C, H, W); ``state=None`` is zeros; no flow warping."""

    def __init__(self, input_size, hidden_size, gru_bias_init=0.0):
        super().__init__()
        self.input_size = input_size
        self.hidden_size = hidden_size
        self.gru_bias_init = gru_bias_init
        self.conv_update = nn.Conv2d(input_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_reset = nn.Conv2d(input_size + hidden_size, hidden_size, kernel_size=3, bias=True, padding=1)
        self.conv_state_tilde = ConvBlock(input_size + hidden_size, hidden_size, kernel_size=3, bias=False)

    def forward(self, x, state=None, flow=None, mode="bilinear"):
        assert flow is None, "the oracle has no flow warping"
        b, timesteps, _, h, w = x.size()
        rnn_state = torch.zeros(b, self.hidden_size, h, w, device=x.device, dtype=x.dtype) if state is None else state
        rnn_output = []
        for t in range(timesteps):
            rnn_state = self.gru_cell(x[:, t], rnn_state)
            rnn_output.append(rnn_state)
        return torch.stack(rnn_output, dim=1)

    def gru_cell(self, x, state):
        x_and_state = torch.cat([x, state], dim=1)
        update_gate = torch.sigmoid(self.conv_update(x_and_state) + self.gru_bias_init)
        reset_gate = torch.sigmoid(self.conv_reset(x_and_state) + self.gru_bias_init)
        state_tilde = self.conv_state_tilde(torch.cat([x, (1.0 - reset_gate) * state], dim=1))
        return (1.0 - update_gate) * state + update_gate * state_tilde


class FuturePrediction(nn.Module):
    """[SpatialGRU, [Bottleneck] x n_res_layers] x n_gru_blocks; every GRU starts from the same hidden state."""

    def __init__(self, in_channels, latent_dim, n_gru_blocks=3, n_res_layers=3):
        super().__init__()
        self.n_gru_blocks = n_gru_blocks
        self.spatial_grus = nn.ModuleList(
            [SpatialGRU(latent_dim if i == 0 else in_channels, in_channels) for i in range(n_gru_blocks)])
        self.res_blocks = nn.ModuleList(
            [nn.Sequential(*[Bottleneck(in_channels) for _ in range(n_res_layers)]) for _ in range(n_gru_blocks)])

    def forward(self, x, hidden_state):
        for i in range(self.n_gru_blocks):
            x = self.spatial_grus[i](x, hidden_state, flow=None)
            b, n_future, c, h, w = x.shape
            x = self.res_blocks[i](x.view(b * n_future, c, h, w))
            x = x.view(b, n_future, c, h, w)
        return x
