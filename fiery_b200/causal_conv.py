"""The temporal model's causal convolutions on the tensor cores (``CausalConv3d``, fiery/layers/temporal.py:65-85).

A reference ``CausalConv3d`` is a zero pad (``kt - 1`` frames in front, one pixel around the map), a bias-free ``Conv3d`` with kernel
(kt, 3, 3), a ``BatchNorm3d`` and a ``ReLU``.  ``torch.ops.fiery_b200.causal_conv3d`` (registered below through fiery_b200/ops.py;
kernels in csrc/causal_conv.cu) computes the pad and the convolution in one pass over a contiguous (b, C, s, X, Y) tensor, without a
padded copy; both gradients run on the tensor cores too, and the weight gradient is bit-reproducible.

``TensorCoreCausalConv3d.from_module(m)`` adopts the reference module's children under the same names (``state_dict`` keys are
unchanged) and replaces only the pad and the convolution; BatchNorm and ReLU stay the module's own, called through
``batch_norm.norm_act`` (one fused apply once ``install.use_fused_batch_norm`` has swapped the norm).
``install.use_tensor_core_causal_convs`` swaps it into a model.  No CPU path.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import _lib
from ._lib import _require_cuda, f32
from .batch_norm import norm_act
from .ops import _register_conv

MAX_CHANNELS = 64


def unsupported_reason(in_channels: int, out_channels: int, kt: int, grid_y: Optional[int] = None) -> Optional[str]:
    """None if the kernels take these shapes, else the reason (the limits of include/fiery_b200.h)."""
    if not 1 <= in_channels <= MAX_CHANNELS:
        return f"in_channels = {in_channels} (the kernels take 1..{MAX_CHANNELS})"
    if not 1 <= out_channels <= MAX_CHANNELS:
        return f"out_channels = {out_channels} (the kernels take 1..{MAX_CHANNELS})"
    if kt not in (1, 2):
        return f"kernel ({kt}, 3, 3) (the kernels take kt = 1 or 2)"
    if grid_y is not None and grid_y % 4:
        return f"Y = {grid_y} map columns (the kernels need a multiple of 4: 16-byte TMA row pitch)"
    return None


def _desc(shape, out_channels: int, kt: int) -> _lib.CausalConv3dDesc:
    b, c, s, h, w = shape
    d = _lib.CausalConv3dDesc()
    d.batch, d.frames, d.grid_x, d.grid_y, d.in_channels, d.out_channels, d.kt = b, s, h, w, c, out_channels, kt
    return d


def pack_weights(weights, in_channels: int) -> torch.Tensor:
    """[(C_out, C_in, kt, 3, 3) weight] -> the uint8 device pack the forward and the input gradient take."""
    (weight,) = weights
    _require_cuda(weight, "weight")
    lib = _lib.load()
    w = f32(weight.detach())
    c_out, c_in, kt = int(w.shape[0]), int(w.shape[1]), int(w.shape[2])
    d = _desc((0, c_in, 0, 1, 4), c_out, kt)
    n = int(lib.fiery_causal_conv3d_packed_bytes(d))
    if n == 0 or tuple(w.shape[3:]) != (3, 3):
        raise _lib.FieryError(f"causal conv: weight {tuple(w.shape)} is not supported: "
                              f"{unsupported_reason(c_in, c_out, kt) or 'kernel must be (kt, 3, 3)'}")
    out = torch.empty(n, dtype=torch.uint8, device=w.device)
    _lib.call("fiery_causal_conv3d_pack_weights", w.device, d, w.data_ptr(), out.data_ptr())
    return out


def _packed(weight: torch.Tensor) -> torch.Tensor:
    return _lib.packed(pack_weights, [weight], int(weight.shape[1]))


def _check(x_shape, weight: torch.Tensor) -> int:
    c_out, c_in, kt = int(weight.shape[0]), int(weight.shape[1]), int(weight.shape[2])
    if x_shape[1] != c_in or tuple(weight.shape[3:]) != (3, 3):
        raise ValueError(f"causal conv: x {tuple(x_shape)} and weight {tuple(weight.shape)} do not match")
    reason = unsupported_reason(c_in, c_out, kt, int(x_shape[4]))
    if reason is not None:
        raise _lib.FieryError(f"causal conv: {reason}")
    return kt


def conv_forward(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """x (b, C_in, s, X, Y) any float dtype and strides; weight (C_out, C_in, kt, 3, 3).  Returns the contiguous fp32
    (b, C_out, s, X, Y) output of the causal pad + Conv3d."""
    _require_cuda(x, "x")
    kt = _check(x.shape, weight)
    xs = f32(x)
    b, _, s, h, w = xs.shape
    y = torch.empty((b, weight.shape[0], s, h, w), dtype=torch.float32, device=x.device)
    packed = _packed(weight)
    _lib.call("fiery_causal_conv3d_forward", x.device, _desc(xs.shape, int(weight.shape[0]), kt), xs.data_ptr(), packed.data_ptr(),
              y.data_ptr())
    return y


def conv_backward_data(grad_y: torch.Tensor, x_shape, weight: torch.Tensor) -> torch.Tensor:
    """The input gradient: a contiguous fp32 tensor of x's shape."""
    kt = _check(x_shape, weight)
    g = f32(grad_y)
    gx = torch.empty(tuple(x_shape), dtype=torch.float32, device=g.device)
    packed = _packed(weight)
    _lib.call("fiery_causal_conv3d_backward_data", g.device, _desc(tuple(x_shape), int(weight.shape[0]), kt), g.data_ptr(),
              packed.data_ptr(), gx.data_ptr())
    return gx


def backward_weight_workspace_bytes(x_shape, out_channels: int, kt: int) -> int:
    """Bytes of device workspace the weight gradient uses (host-only answer; 0 for 0 frames or unsupported shapes)."""
    return int(_lib.load().fiery_causal_conv3d_backward_weight_workspace_bytes(_desc(tuple(x_shape), out_channels, kt)))


def conv_backward_weight(grad_y: torch.Tensor, x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """The weight gradient, fp32 of the weight's shape; bit-reproducible (fixed summation order, no atomics)."""
    lib = _lib.load()
    kt = _check(x.shape, weight)
    xs, g = f32(x), f32(grad_y)
    d = _desc(xs.shape, int(weight.shape[0]), kt)
    ws = _lib.workspace(lib.fiery_causal_conv3d_backward_weight_workspace_bytes(d), x.device)
    gw = torch.empty(tuple(weight.shape), dtype=torch.float32, device=x.device)
    _lib.call("fiery_causal_conv3d_backward_weight", x.device, d, xs.data_ptr(), g.data_ptr(), gw.data_ptr(), ws.data_ptr())
    return gw


# ``torch.ops.fiery_b200.causal_conv3d(x, weight)``: x (b, C_in, s, X, Y), Y % 4 == 0; weight (C_out, C_in, kt, 3, 3), kt 1 or 2 ->
# the contiguous (b, C_out, s, X, Y) fp32 ``Conv3d(ConstantPad3d((1, 1, 1, 1, kt - 1, 0))(x))``; a non-contiguous or 16-bit x is read
# from a contiguous fp32 copy.  ``causal_conv3d_backward``: grad_x of x's shape and dtype, contiguous; grad_weight bit-reproducible
# (no atomics).  The gradients are looked up by name when the operator runs, so a wrapper put in their place sees every launch.
_register_conv(
    "causal_conv3d",
    forward=conv_forward,
    grad_layout=f32,
    grad_input=lambda g, x, weight: conv_backward_data(g, tuple(x.shape), weight),
    grad_weight=lambda g, x, weight: conv_backward_weight(g, x, weight),
    fake_output=lambda x, weight: x.new_empty((x.shape[0], weight.shape[0], *x.shape[2:]), dtype=torch.float32),
    fake_grad_input=lambda x: x.new_empty(x.shape))


# ------------------------------------------------------------------------------------------------------------------------------
# module
# ------------------------------------------------------------------------------------------------------------------------------
def module_reason(m) -> Optional[str]:
    """None if ``m`` (a reference CausalConv3d) is covered by the kernels, else the reason.  The map width is checked at call time."""
    pad, conv = getattr(m, "pad", None), getattr(m, "conv", None)
    if not isinstance(conv, nn.Conv3d) or not isinstance(pad, nn.ConstantPad3d):
        return f"{type(m).__name__} does not have the CausalConv3d structure"
    kt = conv.kernel_size[0]
    if not (conv.kernel_size[1:] == (3, 3) and conv.stride == (1, 1, 1) and conv.padding == (0, 0, 0) and conv.dilation == (1, 1, 1)
            and conv.groups == 1 and conv.bias is None and conv.padding_mode == "zeros"):
        return f"{conv} is not a bias-free (kt, 3, 3) Conv3d with stride 1 and dilation 1"
    if tuple(pad.padding) != (1, 1, 1, 1, kt - 1, 0) or pad.value != 0:
        return f"pad {tuple(pad.padding)} is not the causal zero pad of a ({kt}, 3, 3) kernel"
    return unsupported_reason(conv.in_channels, conv.out_channels, kt)


class TensorCoreCausalConv3d(nn.Module):
    """Drop-in for a reference ``CausalConv3d`` whose pad and convolution run on the tensor cores
    (``torch.ops.fiery_b200.causal_conv3d``).  It holds the reference module's ``pad``, ``conv``, ``norm`` and ``activation`` under the
    same names (``state_dict`` keys are unchanged, the Parameters are shared) and looks them up at call time, so
    ``SyncBatchNorm.convert_sync_batchnorm`` works before or after the swap.  A map whose width Y is not a multiple of 4 runs the
    reference's pad and Conv3d, with one warning."""

    def __init__(self, m):
        super().__init__()
        self.pad = m.pad
        self.conv = m.conv
        self.norm = m.norm
        self.activation = m.activation

    @classmethod
    def from_module(cls, m) -> "TensorCoreCausalConv3d":
        reason = module_reason(m)
        if reason is not None:
            raise ValueError(f"CausalConv3d not covered by the tensor-core kernels: {reason}")
        return cls(m)

    def forward(self, *inputs):
        (x,) = inputs
        width = x.shape[4]
        if width % 4:
            _lib.warn_once(("causal_width", width), f"fiery_b200: CausalConv3d input of Y = {width} map columns is not covered by the "
                           "tensor-core kernels (they need a multiple of 4); it runs as the reference's pad and Conv3d")
            y = self.conv(self.pad(x))
        else:
            y = torch.ops.fiery_b200.causal_conv3d(x, self.conv.weight)
        return norm_act(self.norm, self.activation, y)
