"""First BEV convolution on the tensor cores, behind the reference's module interface (SURVEY.md section 8f, next-2).

``Decoder.first_conv`` (fiery/models/decoder.py:11,59) is ``nn.Conv2d(64, 64, kernel_size=7, stride=2, padding=3, bias=False)``,
followed by ``bn1`` and ``relu`` (decoder.py:60-61).  ``FirstConv`` carries the same parameter (``weight`` (64, 64, 7, 7), so a
reference ``state_dict`` entry ``first_conv.weight`` loads unchanged) and runs the layer as a wgmma implicit GEMM
(fiery_b200/csrc/bev_conv.cu: TF32 operands, fp32 accumulation).  It takes the lift's channel-last BEV directly
(``LiftSplat(output_layout="channels_last")``), so the lift's NCHW layout pass is not on this path.

Training: the backward (fiery_b200/csrc/bev_conv_bwd.cu) computes the input and weight gradients on the tensor cores too, on the
same channel-last layout, bit-reproducibly (no atomics).  ``FirstConv(bn=None)`` -- with or without ``relu`` -- trains through the
``torch.ops.fiery_b200.first_conv`` operator (registered below through fiery_b200/ops.py) whenever grad is enabled;
``install.use_tensor_core_first_conv`` swaps it into a ``Fiery`` model, leaving ``bn1`` and ``relu`` to the reference's modules.
With ``bn`` given the module folds bn1 from its running statistics into the kernel's epilogue: that form is for inference only and
has no backward.  No CPU path.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import _lib
from ._lib import _require_cuda
from .ops import _register_conv


def first_conv_forward(x: torch.Tensor, packed_weight: torch.Tensor, scale: Optional[torch.Tensor] = None,
                       shift: Optional[torch.Tensor] = None, relu: bool = False) -> torch.Tensor:
    """x: (B, 64, H, W) fp32 with channels-last strides (physical (B, H, W, 64)); packed_weight (49, 64, 64) from ``pack_weight``;
    returns (B, 64, Ho, Wo) fp32, channels-last strides, ``relu(conv(x) * scale + shift)`` (scale/shift/relu optional)."""
    _require_cuda(x, "x")
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
    _lib.call("fiery_bev_first_conv_forward", x.device, B, H, W, xs.data_ptr(), packed_weight.data_ptr(),
              sc.data_ptr() if sc is not None else 0, sh.data_ptr() if sh is not None else 0, 1 if relu else 0, store.data_ptr())
    return store.permute(0, 3, 1, 2)


def pack_weight(weight: torch.Tensor) -> torch.Tensor:
    """(64, 64, 7, 7) conv weight -> (49, 64, 64) = (tap, out, in), the K-major B operand of every tap (device kernel)."""
    _require_cuda(weight, "weight")
    if tuple(weight.shape) != (64, 64, 7, 7):
        raise ValueError(f"first_conv weight must be (64, 64, 7, 7), got {tuple(weight.shape)}")
    w = weight.detach().float().contiguous()
    out = torch.empty((49, 64, 64), dtype=torch.float32, device=w.device)
    _lib.call("fiery_bev_conv_pack_weights", w.device, w.data_ptr(), out.data_ptr())
    return out


def pack_weight_transposed(weight: torch.Tensor) -> torch.Tensor:
    """(64, 64, 7, 7) conv weight -> (49, 64, 64) = (tap, in, out), TF32-rounded: the B operand of the input gradient (device kernel)."""
    _require_cuda(weight, "weight")
    if tuple(weight.shape) != (64, 64, 7, 7):
        raise ValueError(f"first_conv weight must be (64, 64, 7, 7), got {tuple(weight.shape)}")
    w = weight.detach().float().contiguous()
    out = torch.empty((49, 64, 64), dtype=torch.float32, device=w.device)
    _lib.call("fiery_bev_conv_pack_weights_transposed", w.device, w.data_ptr(), out.data_ptr())
    return out


def _channels_last_f32(t: torch.Tensor) -> torch.Tensor:
    t = t.float() if t.dtype != torch.float32 else t
    return t if t.permute(0, 2, 3, 1).is_contiguous() else t.contiguous(memory_format=torch.channels_last)


def first_conv_backward_data(grad_y: torch.Tensor, packed_weight_t: torch.Tensor, height: int, width: int) -> torch.Tensor:
    """grad_y (B, 64, Ho, Wo) in any layout (converted to channels-last fp32 once if needed); packed_weight_t (49, 64, 64) from
    ``pack_weight_transposed``; returns grad_x (B, 64, height, width) fp32 with channels-last strides."""
    _require_cuda(grad_y, "grad_y")
    B = grad_y.shape[0]
    if grad_y.dim() != 4 or grad_y.shape[1] != 64 or tuple(grad_y.shape[2:]) != ((height - 1) // 2 + 1, (width - 1) // 2 + 1):
        raise ValueError(f"grad_y {tuple(grad_y.shape)} does not match an input of {height}x{width}")
    g = _channels_last_f32(grad_y)
    store = torch.empty((B, height, width, 64), dtype=torch.float32, device=g.device)
    _lib.call("fiery_bev_first_conv_backward_data", g.device, B, height, width, g.data_ptr(), packed_weight_t.data_ptr(),
              store.data_ptr())
    return store.permute(0, 3, 1, 2)


def backward_weight_workspace_bytes(n_frames: int, height: int, width: int) -> int:
    """Bytes of device workspace ``first_conv_backward_weight`` uses (host-only answer)."""
    return int(_lib.load().fiery_bev_first_conv_backward_weight_workspace_bytes(n_frames, height, width))


def first_conv_backward_weight(x: torch.Tensor, grad_y: torch.Tensor, workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x (B, 64, H, W), grad_y (B, 64, Ho, Wo), any layout and floating dtype (converted to channels-last fp32 once if needed);
    returns the weight gradient (64, 64, 7, 7) fp32, bit-reproducible.  ``workspace``: a uint8 device tensor of at least
    ``backward_weight_workspace_bytes`` bytes to use instead of a fresh one."""
    _require_cuda(x, "x")
    if x.dim() != 4 or x.shape[1] != 64:
        raise ValueError(f"x must be (B, 64, H, W), got {tuple(x.shape)}")
    B, _, H, W = x.shape
    if tuple(grad_y.shape) != (B, 64, (H - 1) // 2 + 1, (W - 1) // 2 + 1):
        raise ValueError(f"grad_y {tuple(grad_y.shape)} does not match x {tuple(x.shape)}")
    xs, g = _channels_last_f32(x), _channels_last_f32(grad_y)
    need = backward_weight_workspace_bytes(B, H, W)
    if workspace is None or workspace.numel() < need:
        workspace = _lib.workspace(need, x.device)
    out = torch.empty((64, 64, 7, 7), dtype=torch.float32, device=x.device)
    _lib.call("fiery_bev_first_conv_backward_weight", x.device, B, H, W, xs.data_ptr(), g.data_ptr(), out.data_ptr(),
              workspace.data_ptr())
    return out


# ``torch.ops.fiery_b200.first_conv(x, weight)``: x (B, 64, H, W), any layout and floating dtype -> (B, 64, Ho, Wo) fp32 with
# channels-last strides.  ``first_conv_backward``: grad_x of x's shape and dtype with channels-last strides (so a
# ``LiftSplat(output_layout="channels_last")`` upstream takes its NHWC backward route); grad_weight bit-reproducible (no atomics).
# grad_y is converted to channels-last fp32 once, shared by both gradients.  The weight's packs come from ``_lib.packed``, the
# transposed one only when the input gradient is asked for.
_register_conv(
    "first_conv",
    forward=lambda x, weight: first_conv_forward(x, _lib.packed(pack_weight, weight)),
    grad_layout=_channels_last_f32,
    grad_input=lambda g, x, weight: first_conv_backward_data(g, _lib.packed(pack_weight_transposed, weight), x.shape[2], x.shape[3]),
    grad_weight=lambda g, x, weight: first_conv_backward_weight(x, g),
    fake_output=lambda x, weight: x.new_empty((x.shape[0], (x.shape[2] - 1) // 2 + 1, (x.shape[3] - 1) // 2 + 1, 64),
                                              dtype=torch.float32).permute(0, 3, 1, 2),
    fake_grad_input=lambda x: x.new_empty((x.shape[0], x.shape[2], x.shape[3], x.shape[1])).permute(0, 3, 1, 2))


class FirstConv(nn.Module):
    """Drop-in for ``Decoder.first_conv`` (+ ``bn1`` + ``relu`` when given).  Without ``bn`` it trains: whenever grad is enabled the
    forward runs through the ``fiery_b200::first_conv`` operator, whose backward computes the input and weight gradients on the tensor
    cores, and ``relu`` (if asked) is applied after it by ``torch.relu``; the forward values are those of the fused inference kernel.
    With ``bn`` (bn1 folded from its running statistics into the epilogue) it is eval-only: ``.train()`` mode raises, and no gradient
    flows through it.  ``FirstConv.from_decoder(decoder)`` and ``FirstConv.from_conv(conv)`` adopt the reference module's parameters
    (shared, not copied)."""

    def __init__(self, bn: Optional[nn.BatchNorm2d] = None, relu: bool = False):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(64, 64, 7, 7))
        nn.init.kaiming_normal_(self.weight, mode="fan_out", nonlinearity="relu")
        self.bn, self.relu = bn, relu

    @classmethod
    def from_decoder(cls, decoder, fuse_bn_relu: bool = True) -> "FirstConv":
        m = cls(bn=decoder.bn1 if fuse_bn_relu else None, relu=fuse_bn_relu)
        m.weight = decoder.first_conv.weight
        return m

    @classmethod
    def from_conv(cls, conv: nn.Conv2d) -> "FirstConv":
        """The trainable form (``bn=None``) of ``Decoder.first_conv`` = ``conv``, sharing its weight Parameter."""
        m = cls()
        m.weight = conv.weight
        return m

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
        if self.bn is None and torch.is_grad_enabled():
            y = torch.ops.fiery_b200.first_conv(x, self.weight)
            return torch.relu(y) if self.relu else y
        with torch.no_grad():
            return first_conv_forward(x, _lib.packed(pack_weight, self.weight), scale, shift, self.relu)
