"""First BEV convolution on the tensor cores, behind the reference's module interface (SURVEY.md section 8f, next-2).

``Decoder.first_conv`` (fiery/models/decoder.py:11,59) is ``nn.Conv2d(64, 64, kernel_size=7, stride=2, padding=3, bias=False)``,
followed by ``bn1`` and ``relu`` (decoder.py:60-61).  ``FirstConv`` carries the same parameter (``weight`` (64, 64, 7, 7), so a
reference ``state_dict`` entry ``first_conv.weight`` loads unchanged) and runs the layer as a wgmma implicit GEMM
(fiery_b200/csrc/bev_conv.cu: TF32 operands, fp32 accumulation).  It takes the lift's channel-last BEV directly
(``LiftSplat(output_layout="channels_last")``), so the lift's NCHW layout pass is not on this path.

Inference op: no backward (training keeps ``nn.Conv2d``; the reference trains this layer under cuDNN).  No CPU path.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import _lib
from .geometry import _require_cuda, _stream_ptr


def first_conv_forward(x: torch.Tensor, packed_weight: torch.Tensor, scale: Optional[torch.Tensor] = None,
                       shift: Optional[torch.Tensor] = None, relu: bool = False) -> torch.Tensor:
    """x: (B, 64, H, W) fp32 with channels-last strides (physical (B, H, W, 64)); packed_weight (49, 64, 64) from ``pack_weight``;
    returns (B, 64, Ho, Wo) fp32, channels-last strides, ``relu(conv(x) * scale + shift)`` (scale/shift/relu optional)."""
    _require_cuda(x, "x")
    lib = _lib.load()
    if x.dim() != 4 or x.shape[1] != 64:
        raise ValueError(f"x must be (B, 64, H, W), got {tuple(x.shape)}")
    B, C, H, W = x.shape
    xs = x.float() if x.dtype != torch.float32 else x
    if not xs.permute(0, 2, 3, 1).is_contiguous():
        xs = xs.contiguous(memory_format=torch.channels_last)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    store = torch.empty((B, Ho, Wo, 64), dtype=torch.float32, device=x.device)
    sc = scale.float().contiguous() if scale is not None else None
    sh = shift.float().contiguous() if shift is not None else None
    with torch.cuda.device(x.device):
        _lib.check(lib.fiery_bev_first_conv_forward(B, H, W, xs.data_ptr(), packed_weight.data_ptr(),
                                                    sc.data_ptr() if sc is not None else 0, sh.data_ptr() if sh is not None else 0,
                                                    1 if relu else 0, store.data_ptr(), _stream_ptr(x.device)),
                   "fiery_bev_first_conv_forward")
    return store.permute(0, 3, 1, 2)


def pack_weight(weight: torch.Tensor) -> torch.Tensor:
    """(64, 64, 7, 7) conv weight -> (49, 64, 64) = (tap, out, in), the K-major B operand of every tap (device kernel)."""
    _require_cuda(weight, "weight")
    if tuple(weight.shape) != (64, 64, 7, 7):
        raise ValueError(f"first_conv weight must be (64, 64, 7, 7), got {tuple(weight.shape)}")
    lib = _lib.load()
    w = weight.detach().float().contiguous()
    out = torch.empty((49, 64, 64), dtype=torch.float32, device=w.device)
    with torch.cuda.device(w.device):
        _lib.check(lib.fiery_bev_conv_pack_weights(w.data_ptr(), out.data_ptr(), _stream_ptr(w.device)), "fiery_bev_conv_pack_weights")
    return out


class FirstConv(nn.Module):
    """Drop-in for ``Decoder.first_conv`` (+ ``bn1`` + ``relu`` when given) in eval mode.  ``FirstConv.from_decoder(decoder)``
    adopts the reference module's parameters (shared, not copied)."""

    def __init__(self, bn: Optional[nn.BatchNorm2d] = None, relu: bool = False):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(64, 64, 7, 7))
        nn.init.kaiming_normal_(self.weight, mode="fan_out", nonlinearity="relu")
        self.bn, self.relu = bn, relu
        self._packed = None

    @classmethod
    def from_decoder(cls, decoder, fuse_bn_relu: bool = True) -> "FirstConv":
        m = cls(bn=decoder.bn1 if fuse_bn_relu else None, relu=fuse_bn_relu)
        m.weight = decoder.first_conv.weight
        return m

    def _packed_weight(self) -> torch.Tensor:
        key = (self.weight.data_ptr(), self.weight._version, str(self.weight.device))
        if self._packed is None or self._packed[0] != key:
            self._packed = (key, pack_weight(self.weight))
        return self._packed[1]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.training and self.bn is not None:
            raise RuntimeError("FirstConv folds bn1 with its running statistics: call .eval() (training keeps nn.Conv2d + BatchNorm2d)")
        scale = shift = None
        if self.bn is not None:                                   # y = (conv - mean) / sqrt(var + eps) * gamma + beta
            inv = torch.rsqrt(self.bn.running_var.float() + self.bn.eps)
            g = self.bn.weight.float() if self.bn.affine else torch.ones_like(inv)
            bta = self.bn.bias.float() if self.bn.affine else torch.zeros_like(inv)
            scale = g * inv
            shift = bta - self.bn.running_mean.float() * scale
        with torch.no_grad():
            return first_conv_forward(x, self._packed_weight(), scale, shift, self.relu)
