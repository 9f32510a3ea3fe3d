"""The decoder's output heads on the project's kernels (fiery/models/decoder.py:24-50).

Each head is ``Conv2d(C, C, 3, padding 1, bias=False) -> BatchNorm2d(C) -> ReLU -> Conv2d(C, n, 1)`` with a bias (the center head adds a
``Sigmoid``), on the decoder's full-resolution map.  The 3x3 stays cuDNN's (``F.conv2d`` with the head's own weight); everything after
it runs as ``torch.ops.fiery_b200.output_head`` (registered in fiery_b200/ops.py; csrc/output_head.cu): the norm's statistics, then
the 1x1 on the tensor cores with the norm and ReLU applied as it reads y and the bias added in its epilogue.  relu(bn(y)) never exists
in memory; the backward recomputes the 1x1's input gradient from grad_out (n <= 8 terms) in its two passes over y and writes dy only.
Everything is bit-reproducible.

``FusedOutputHead.from_module(head)`` adopts the head's children (``state_dict`` keys unchanged) and looks them up at call time;
``install.use_tensor_core_output_heads`` swaps it into a model's decoder.  No CPU path.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from ._lib import _require_cuda, f32
from .batch_norm import update_running_stats

MAX_CHANNELS = 128
MAX_OUTPUTS = 8


def unsupported_reason(channels: int, n_out: int, pixels: Optional[int] = None) -> Optional[str]:
    """None if the kernels take these shapes, else the reason (the limits of include/fiery_b200.h)."""
    if not 1 <= channels <= MAX_CHANNELS:
        return f"{channels} channels (the kernels take 1..{MAX_CHANNELS})"
    if not 1 <= n_out <= MAX_OUTPUTS:
        return f"{n_out} outputs (the kernels take 1..{MAX_OUTPUTS})"
    if pixels is not None and pixels % 4:
        return f"H * W = {pixels} pixels (the kernels need a multiple of 4: 16-byte TMA plane pitch)"
    return None


def desc(maps: int, h: int, w: int, channels: int, n_out: int, training: bool = True, eps: float = 1e-5) -> _lib.OutputHeadDesc:
    d = _lib.OutputHeadDesc()
    d.maps, d.grid_x, d.grid_y, d.channels, d.n_out, d.training, d.eps = maps, h, w, channels, n_out, int(training), float(eps)
    return d


def workspace_bytes(maps: int, h: int, w: int, channels: int, n_out: int) -> Tuple[int, int, int]:
    """(pack, forward workspace, backward workspace) bytes from the C ABI (host-only; 0s for shapes outside the limits)."""
    lib = _lib.load()
    d = desc(maps, h, w, channels, n_out)
    return (int(lib.fiery_output_head_packed_bytes(d)), int(lib.fiery_output_head_forward_workspace_bytes(d)),
            int(lib.fiery_output_head_backward_workspace_bytes(d)))


def pack_weights(weights) -> torch.Tensor:
    """[W1 (n, C, 1, 1), b1 (n,)] -> the uint8 device pack of the 1x1 (W1 with b1 as its last column)."""
    w1, b1 = weights
    _require_cuda(w1, "weight")
    n, c = int(w1.shape[0]), int(w1.shape[1])
    if tuple(w1.shape) != (n, c, 1, 1) or tuple(b1.shape) != (n,):
        raise ValueError(f"output head: weights {tuple(w1.shape)}, {tuple(b1.shape)} are not (n, C, 1, 1), (n,)")
    reason = unsupported_reason(c, n)
    if reason is not None:
        raise _lib.FieryError(f"output head: {reason}")
    stacked = torch.cat([f32(w1.detach()).reshape(n, c), f32(b1.detach()).reshape(n, 1)], 1).contiguous()
    d = desc(1, 1, 4, c, n)
    out = torch.empty(int(_lib.load().fiery_output_head_packed_bytes(d)), dtype=torch.uint8, device=w1.device)
    _lib.call("fiery_output_head_pack_weights", w1.device, d, stacked.data_ptr(), out.data_ptr())
    return out


def _packed(w1: torch.Tensor, b1: torch.Tensor) -> torch.Tensor:
    return _lib.packed(pack_weights, [w1, b1])


def _ptr(t: Optional[torch.Tensor]) -> int:
    return t.data_ptr() if t is not None else 0


def _aligned_f32(t: torch.Tensor) -> torch.Tensor:
    """t as a contiguous, 16-byte aligned fp32 tensor: t itself when it is one, else a copy."""
    if t.dtype == torch.float32 and t.is_contiguous() and t.data_ptr() % 16 == 0:
        return t
    return t.to(torch.float32, memory_format=torch.contiguous_format, copy=True)


def _check(y: torch.Tensor, w1: torch.Tensor) -> Tuple[int, int, int, int, int]:
    if y.dim() != 4 or y.shape[1] != w1.shape[1]:
        raise ValueError(f"output head: y {tuple(y.shape)} is not (N, {int(w1.shape[1])}, H, W)")
    m, c, h, w = (int(v) for v in y.shape)
    n = int(w1.shape[0])
    reason = unsupported_reason(c, n, h * w)
    if reason is not None:
        raise _lib.FieryError(f"output head: {reason}")
    return m, c, h, w, n


def forward(y, w1, b1, bn_weight, bn_bias, running_mean, running_var, training: bool, eps: float):
    """(out, mean, var): out (N, n, H, W) = conv1x1(relu(bn(y)), W1, b1) fp32 on y (N, C, H, W), and the (C,) fp32 mean and biased var
    the norm used (the batch's when ``training``, else copies of ``running_mean`` / ``running_var``)."""
    _require_cuda(y, "y")
    m, c, h, w, n = _check(y, w1)
    if not training and (running_mean is None or running_var is None):
        raise ValueError("output head: eval mode needs running_mean and running_var")
    ys = _aligned_f32(y)
    bn_w, bn_b, rm, rv = (f32(p.detach()) if p is not None else None for p in (bn_weight, bn_bias, running_mean, running_var))
    d = desc(m, h, w, c, n, training, eps)
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=y.device)  # noqa: E731
    out, mean, var = new(m, n, h, w), new(c), new(c)
    ws = _lib.workspace(_lib.load().fiery_output_head_forward_workspace_bytes(d), y.device)
    _lib.call("fiery_output_head_forward", y.device, d, ys.data_ptr(), _packed(w1, b1).data_ptr(), _ptr(bn_w), _ptr(bn_b), _ptr(rm),
              _ptr(rv), out.data_ptr(), mean.data_ptr(), var.data_ptr(), ws.data_ptr())
    return out, mean, var


def backward(grad_out, y, mean, var, w1, b1, bn_weight, bn_bias, training: bool, eps: float, need: List[bool]):
    """The gradients of ``forward`` in fp32, [grad_y, grad_bn_weight, grad_bn_bias, grad_W1 (n, C, 1, 1), grad_b1], None where ``need``
    (5 flags in that order) does not ask or the norm has no such parameter."""
    m, c, h, w, n = _check(y, w1)
    dev = y.device
    ys, go, w1s = _aligned_f32(y), _aligned_f32(grad_out), f32(w1.detach())
    bn_w, bn_b = (f32(p.detach()) if p is not None else None for p in (bn_weight, bn_bias))
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)  # noqa: E731
    gy = new(m, c, h, w) if need[0] else None
    gbw = new(c) if need[1] and bn_weight is not None else None
    gbb = new(c) if need[2] and bn_bias is not None else None
    gw = new(n, c, 1, 1) if need[3] else None
    gb = new(n) if need[4] else None
    d = desc(m, h, w, c, n, training, eps)
    ws = _lib.workspace(_lib.load().fiery_output_head_backward_workspace_bytes(d), dev)
    _lib.call("fiery_output_head_backward", dev, d, go.data_ptr(), ys.data_ptr(), mean.data_ptr(), var.data_ptr(),
              w1s.data_ptr(), _ptr(bn_w), _ptr(bn_b), _ptr(gy), _ptr(gbw), _ptr(gbb), _ptr(gw), _ptr(gb), ws.data_ptr())
    return [gy, gbw, gbb, gw, gb]


# ------------------------------------------------------------------------------------------------------------------------------
# module
# ------------------------------------------------------------------------------------------------------------------------------
def module_reason(head) -> Optional[str]:
    """None if ``head`` (a reference output head) is the structure the kernels cover, else the reason.  The map size is checked at
    call time."""
    if not isinstance(head, nn.Sequential) or tuple(head._modules) not in (("0", "1", "2", "3"), ("0", "1", "2", "3", "4")):
        return f"{type(head).__name__} does not have the output-head structure (3x3 conv, norm, ReLU, 1x1 conv[, Sigmoid])"
    conv, bn, act, conv1 = (head._modules[k] for k in ("0", "1", "2", "3"))
    if not (type(conv) is nn.Conv2d and conv.kernel_size == (3, 3) and conv.bias is None and conv.padding_mode == "zeros"):
        return "the first convolution is not a bias-free, zero-padded 3x3 Conv2d"
    if type(bn) is not nn.BatchNorm2d:
        return f"norm {type(bn).__name__} (the kernels take BatchNorm2d)"
    if bn.num_features != conv.out_channels:
        return f"a norm of {bn.num_features} channels after a {conv.out_channels}-channel convolution"
    if type(act) is not nn.ReLU:
        return f"activation {type(act).__name__} (the kernels take ReLU)"
    if not (type(conv1) is nn.Conv2d and conv1.kernel_size == (1, 1) and conv1.stride == (1, 1) and conv1.padding == (0, 0)
            and conv1.dilation == (1, 1) and conv1.groups == 1 and conv1.bias is not None and conv1.in_channels == bn.num_features):
        return "the last convolution is not a 1x1 Conv2d with a bias over the norm's channels"
    if "4" in head._modules and type(head._modules["4"]) is not nn.Sigmoid:
        return f"a final {type(head._modules['4']).__name__} (the kernels take Sigmoid or nothing)"
    return unsupported_reason(bn.num_features, conv1.out_channels)


class FusedOutputHead(nn.Sequential):
    """Drop-in for a reference output head whose forward is ``F.conv2d`` with the head's 3x3 weight, then
    ``torch.ops.fiery_b200.output_head`` (BatchNorm2d, ReLU and the 1x1 with its bias), then the Sigmoid if the head has one.  It holds
    the head's children under the same keys (``0``, ``1``, ``2``, ``3``, and ``4`` for the sigmoid; ``state_dict`` keys unchanged, the
    Parameters shared) and looks them up at call time.  The norm's running statistics move as ``nn.BatchNorm2d`` moves them (its own
    momentum, or the cumulative average for momentum None).  A CPU input, a map whose H * W is not a multiple of 4, a norm that is not a
    plain BatchNorm2d (a SyncBatchNorm included) or a convolution or activation changed after the swap run the reference's forward, with
    one warning."""

    @classmethod
    def from_module(cls, head) -> "FusedOutputHead":
        reason = module_reason(head)
        if reason is not None:
            raise ValueError(f"output head not covered by the kernels: {reason}")
        return cls(OrderedDict(head._modules))

    def _call_reason(self, x) -> Optional[str]:
        if not x.is_cuda:
            return "a CPU input"
        if x.dim() != 4:
            return f"a {x.dim()}-D input (the kernels take (N, C, H, W))"
        reason = module_reason(self)
        if reason is not None:
            return reason
        if (x.shape[2] * x.shape[3]) % 4:
            return f"H * W = {x.shape[2] * x.shape[3]} pixels (the kernels need a multiple of 4)"
        return None

    def forward(self, x):
        reason = self._call_reason(x)
        if reason is not None:
            _lib.warn_once(("output_head", reason), f"fiery_b200: output head call not covered by the kernels ({reason}); it runs the "
                           "reference's forward")
            return super().forward(x)
        conv, bn, conv1 = self._modules["0"], self._modules["1"], self._modules["3"]
        y = F.conv2d(x, conv.weight, None, conv.stride, conv.padding, conv.dilation, conv.groups)
        batch_stats = bn.training or (bn.running_mean is None and bn.running_var is None)
        out, mean, var = torch.ops.fiery_b200.output_head(y, conv1.weight, conv1.bias, bn.weight, bn.bias,
                                                          None if batch_stats else bn.running_mean,
                                                          None if batch_stats else bn.running_var, batch_stats, float(bn.eps))
        if batch_stats:
            update_running_stats(bn, mean, var, y.shape[0] * y.shape[2] * y.shape[3])
        if "4" in self._modules:
            out = self._modules["4"](out)
        return out


from . import ops as _ops  # noqa: E402,F401  (registers torch.ops.fiery_b200.output_head)
