"""``Encoder.depth_layer`` on the tensor cores, behind the reference's module interface (SURVEY.md section 8f, next-3).

The reference builds ``self.depth_layer = nn.Conv2d(upsampling_out_channels=128, C + D, kernel_size=1, padding=0)``
(fiery/models/encoder.py:36) and applies it to the backbone features (encoder.py:96); its output is the head tensor the lift
consumes.  ``DepthLayer`` carries the same parameters (``weight`` (C + D, 128, 1, 1), ``bias`` (C + D,): a reference ``state_dict``
loads unchanged) and runs the layer as a wgmma GEMM (fiery_b200/csrc/depth_layer.cu) that reads the features in the dtype the
backbone emits (fp16 / bf16 under AMP, fp32 otherwise) and writes the **fp32** head tensor directly -- the dtype the lift computes in
(the reference's softmax and outer product run in fp32 under autocast, encoder.py:99-100), so an AMP step needs no widening pass
between the two.  The backward (gradients of features, weight and bias) is one library call, ``aten::convolution_backward``.
No CPU path.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from ._lib import _require_cuda

_DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def pack_weight(weight: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """(n_out, 128, 1, 1) -> the (128, 128) row-major operand of the kernel in the features' dtype, rows >= n_out zero."""
    n_out = weight.shape[0]
    if n_out > 128 or tuple(weight.shape[1:]) != (128, 1, 1):
        raise ValueError(f"weight must be (<= 128, 128, 1, 1), got {tuple(weight.shape)}")
    wp = torch.zeros((128, 128), dtype=dtype, device=weight.device)
    wp[:n_out] = weight.detach().reshape(n_out, 128).to(dtype)
    return wp


def depth_layer_forward(feat: torch.Tensor, weight: torch.Tensor, bias, packed: torch.Tensor = None) -> torch.Tensor:
    """feat (N, 128, h, w) fp32 / fp16 / bf16 contiguous; weight (n_out, 128, 1, 1); bias (n_out,) or None -> (N, n_out, h, w) fp32.
    ``packed``: ``pack_weight(weight, feat.dtype)`` made earlier (the module takes it from ``_lib.packed``)."""
    _require_cuda(feat, "feat")
    if feat.dim() != 4 or feat.shape[1] != 128 or feat.dtype not in _DTYPE_CODE:
        raise ValueError(f"feat must be (N, 128, h, w) in fp32 / fp16 / bf16, got {tuple(feat.shape)} {feat.dtype}")
    n_out = weight.shape[0]
    x = feat.contiguous()
    N, _, h, w = x.shape
    wp = packed if packed is not None else pack_weight(weight, x.dtype)
    if wp.dtype != x.dtype or tuple(wp.shape) != (128, 128) or wp.device != x.device:
        raise ValueError("packed weights must be pack_weight(weight, feat.dtype) on the features' device")
    b = None
    if bias is not None:
        b = bias if (bias.dtype == torch.float32 and bias.is_contiguous()) else bias.detach().float().contiguous()
    out = torch.empty((N, n_out, h, w), dtype=torch.float32, device=x.device)
    _lib.call("fiery_depth_layer_forward", x.device, N, h * w, n_out, x.data_ptr(), _DTYPE_CODE[x.dtype], wp.data_ptr(),
              b.data_ptr() if b is not None else 0, out.data_ptr())
    return out


class _DepthLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, weight, bias, packed):
        if packed is None:
            packed = pack_weight(weight, feat.dtype)
        ctx.save_for_backward(feat, weight, packed)
        ctx.has_bias = bias is not None
        return depth_layer_forward(feat, weight, bias, packed)

    @staticmethod
    def backward(ctx, g):                                  # g (N, n_out, h, w) fp32: the lift's grad_head
        """One library call (``aten::convolution_backward``: cuDNN data- and weight-gradient kernels) in the features' dtype -- what
        the reference's convolution backward runs in under autocast (half operands, fp32 accumulation, loss-scaled gradients).  The
        training step is launch-bound, so the backward is kept to a handful of dispatcher calls."""
        feat, weight, packed = ctx.saved_tensors
        n_out = weight.shape[0]
        dt = feat.dtype
        gh = g.contiguous() if g.dtype == dt else g.to(dt)
        w_dt = packed[:n_out].view(n_out, 128, 1, 1)       # the weights already rounded to the operand type (a view: no kernel)
        mask = [ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.has_bias and ctx.needs_input_grad[2]]
        g_feat, g_w, g_b = torch.ops.aten.convolution_backward(gh, feat, w_dt, [n_out] if ctx.has_bias else None, [1, 1], [0, 0], [1, 1],
                                                               False, [0, 0], 1, mask)
        if g_w is not None and g_w.dtype != weight.dtype:
            g_w = g_w.to(weight.dtype)
        if g_b is not None and g_b.dtype != torch.float32:
            g_b = g_b.float()
        return g_feat, g_w, g_b, None


class DepthLayer(nn.Module):
    """Drop-in for ``Encoder.depth_layer`` (encoder.py:36): same parameter names and shapes as the ``nn.Conv2d`` it replaces."""

    def __init__(self, out_channels: int, in_channels: int = 128, bias: bool = True):
        super().__init__()
        if in_channels != 128 or out_channels > 128:
            raise ValueError("the tensor-core kernel is built for 128 input channels and <= 128 outputs (encoder.py:33-36)")
        conv = nn.Conv2d(in_channels, out_channels, kernel_size=1, padding=0, bias=bias)      # the reference's initialisation
        self.weight, self.bias = conv.weight, conv.bias

    def _packed_weight(self, dtype):
        return _lib.packed(pack_weight, self.weight, dtype)        # re-made after every optimizer step (64 KB)

    @classmethod
    def from_conv(cls, conv: nn.Conv2d) -> "DepthLayer":
        m = cls(conv.out_channels, conv.in_channels, conv.bias is not None)
        m.weight, m.bias = conv.weight, conv.bias          # shared, not copied
        return m

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _DepthLayerFn.apply(x, self.weight, self.bias, self._packed_weight(x.dtype))
