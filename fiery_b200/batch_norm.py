"""The temporal model's BatchNorm3d on the project's kernels, with its ReLU and the block's residual add fused (csrc/batch_norm.cu).

Every norm of a ``TemporalBlock`` (fiery/layers/temporal.py:107-117, 65-85, 256-281) normalizes a (b, C, s, X, Y) fp32 map a kernel
has just written, and all but the projection's are followed by ``nn.ReLU(inplace=True)``; the block ends with ``x + x_residual``.
``torch.ops.fiery_b200.batch_norm_act`` (registered in fiery_b200/ops.py) computes ``relu(batch_norm(x)) + residual`` in one apply
pass after one statistics pass, and its backward needs only x and the (C,) statistics: neither the norm's output nor the ReLU's is
kept.  Both are bit-reproducible (no atomics; the summation order depends on the shape only) and graph-capturable.

``FusedBatchNorm3d`` adopts an ``nn.BatchNorm3d``'s Parameters and buffers (``state_dict`` keys unchanged) and follows
``_BatchNorm.forward``'s rules; ``install.use_fused_batch_norm`` swaps it into a model, and ``norm_act`` is where the swapped temporal
modules call ``activation(norm(y))``.  No CPU path.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn as nn

from . import _lib
from ._lib import _require_cuda, f32, f32_planes


def _desc(x: torch.Tensor, training: bool, relu: bool, eps: float) -> _lib.BatchNormDesc:
    b, c, s, h, w = x.shape
    d = _lib.BatchNormDesc()
    d.batch, d.channels, d.frames, d.pixels = b, c, s, h * w
    d.stride_b, d.stride_c, d.stride_t = x.stride(0), x.stride(1), x.stride(2)
    d.training, d.relu, d.eps = int(training), int(relu), float(eps)
    return d


def _per_channel(t: Optional[torch.Tensor], c: int, name: str) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if tuple(t.shape) != (c,):
        raise ValueError(f"batch norm: {name} has shape {tuple(t.shape)}, expected ({c},)")
    return f32(t.detach())


def _workspace(d: _lib.BatchNormDesc, device: torch.device) -> torch.Tensor:
    return _lib.workspace(_lib.load().fiery_batch_norm_workspace_bytes(d), device)


def _check_count(x_shape, training: bool) -> None:
    b, _, s, h, w = x_shape
    if training and b * s * h * w < 2:
        raise ValueError(f"Expected more than 1 value per channel when training, got input size {torch.Size(x_shape)}")


def forward(x: torch.Tensor, weight: Optional[torch.Tensor], bias: Optional[torch.Tensor], running_mean: Optional[torch.Tensor],
            running_var: Optional[torch.Tensor], residual: Optional[torch.Tensor], training: bool, eps: float,
            relu: bool) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """x (b, C, s, X, Y) any float dtype and strides -> (y, mean, var): y the contiguous fp32 ``relu(batch_norm(x)) + residual`` (ReLU
    when ``relu``, the add when ``residual`` is given), mean and the biased var the (C,) fp32 statistics it normalized with (the
    batch's in training, copies of the running ones in eval).  Nothing is updated in place."""
    _require_cuda(x, "x")
    if x.dim() != 5:
        raise ValueError(f"batch norm: expected a 5-D (b, C, s, X, Y) input, got {tuple(x.shape)}")
    _check_count(x.shape, training)
    xs = f32_planes(x)
    c = int(xs.shape[1])
    w, bs = _per_channel(weight, c, "weight"), _per_channel(bias, c, "bias")
    rm, rv = _per_channel(running_mean, c, "running_mean"), _per_channel(running_var, c, "running_var")
    if not training and (rm is None or rv is None):
        raise ValueError("batch norm: eval mode needs running_mean and running_var")
    if residual is not None and tuple(residual.shape) != tuple(xs.shape):
        raise ValueError(f"batch norm: residual {tuple(residual.shape)} does not match x {tuple(xs.shape)}")
    r = f32(residual) if residual is not None else None
    y = torch.empty(tuple(xs.shape), dtype=torch.float32, device=x.device)
    mean = torch.empty(c, dtype=torch.float32, device=x.device)
    var = torch.empty(c, dtype=torch.float32, device=x.device)
    d = _desc(xs, training, relu, eps)
    ptr = lambda t: t.data_ptr() if t is not None else 0           # noqa: E731
    _lib.call("fiery_batch_norm_forward", x.device, d, xs.data_ptr(), ptr(w), ptr(bs), ptr(rm), ptr(rv), ptr(r), y.data_ptr(),
              mean.data_ptr(), var.data_ptr(), _workspace(d, x.device).data_ptr())
    return y, mean, var


def backward(grad_y: torch.Tensor, x: torch.Tensor, weight: Optional[torch.Tensor], bias: Optional[torch.Tensor], mean: torch.Tensor,
             var: torch.Tensor, training: bool, eps: float, relu: bool, need_input: bool, need_weight: bool, need_bias: bool):
    """(grad_x, grad_weight, grad_bias) of ``forward`` in fp32 (grad_x contiguous), None where not asked for; ``mean`` / ``var`` are
    the forward's outputs, and the weight and bias the forward's, so the ReLU mask is the forward's."""
    xs = f32_planes(x)
    c = int(xs.shape[1])
    g = f32(grad_y)
    w, bs = _per_channel(weight, c, "weight"), _per_channel(bias, c, "bias")
    dx = torch.empty(tuple(xs.shape), dtype=torch.float32, device=x.device) if need_input else None
    dw = torch.empty(c, dtype=torch.float32, device=x.device) if need_weight else None
    db = torch.empty(c, dtype=torch.float32, device=x.device) if need_bias else None
    d = _desc(xs, training, relu, eps)
    ptr = lambda t: t.data_ptr() if t is not None else 0           # noqa: E731
    _lib.call("fiery_batch_norm_backward", x.device, d, xs.data_ptr(), g.data_ptr(), ptr(w), ptr(bs), f32(mean).data_ptr(),
              f32(var).data_ptr(), ptr(dx), ptr(dw), ptr(db), _workspace(d, x.device).data_ptr())
    return dx, dw, db


# ------------------------------------------------------------------------------------------------------------------------------
# module
# ------------------------------------------------------------------------------------------------------------------------------
class FusedBatchNorm3d(nn.BatchNorm3d):
    """Drop-in for an ``nn.BatchNorm3d`` that runs on ``torch.ops.fiery_b200.batch_norm_act``.  It adopts the module's Parameters and
    buffers (the same objects: ``state_dict`` keys are unchanged and optimizers still hold them) and follows ``_BatchNorm.forward``'s
    rules: batch statistics when training or when there are no running statistics, ``num_batches_tracked`` counted, ``momentum=None``
    a cumulative average, the running variance updated with the unbiased variance.  The running statistics are updated on the device
    from the operator's (mean, var), without a host synchronisation, so a step can be captured in a CUDA graph.
    ``forward_act(x, relu, residual)`` is the fused entry.  Being a ``_BatchNorm``, ``SyncBatchNorm.convert_sync_batchnorm`` turns it
    into an (unfused) ``SyncBatchNorm`` holding the same tensors."""

    def __init__(self, bn: nn.BatchNorm3d):
        nn.Module.__init__(self)
        for name in ("num_features", "eps", "momentum", "affine", "track_running_stats"):
            setattr(self, name, getattr(bn, name))
        for name, p in bn._parameters.items():
            self.register_parameter(name, p)
        for name, b in bn._buffers.items():
            self.register_buffer(name, b, persistent=name not in bn._non_persistent_buffers_set)
        self.train(bn.training)

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        return self.forward_act(input, relu=False)

    def forward_act(self, x: torch.Tensor, relu: bool, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``relu(self(x)) + residual`` (the ReLU when ``relu``, the add when ``residual`` is given) in one apply pass; the output is
        contiguous fp32."""
        self._check_input_dim(x)
        batch_stats = self.training or (self.running_mean is None and self.running_var is None)
        y, mean, var = torch.ops.fiery_b200.batch_norm_act(
            x, self.weight, self.bias, None if batch_stats else self.running_mean, None if batch_stats else self.running_var, residual,
            batch_stats, self.eps, relu)
        if batch_stats:
            self.update_running_stats(mean, var, x.numel() // x.shape[1])
        return y

    def update_running_stats(self, mean: torch.Tensor, var: torch.Tensor, n: int) -> None:
        """``update_running_stats(self, mean, var, n)``."""
        update_running_stats(self, mean, var, n)


def update_running_stats(bn: nn.Module, mean: torch.Tensor, var: torch.Tensor, n: int) -> None:
    """``_BatchNorm.forward``'s bookkeeping on the norm ``bn`` for a batch of n values per channel with this mean and biased variance,
    as device tensor operations: nothing in eval or without tracked statistics, else ``num_batches_tracked += 1`` and each running
    statistic moved toward the batch's by the momentum (``1 / num_batches_tracked`` when the momentum is None), the variance as the
    unbiased n / (n - 1) var.  ``FusedBatchNorm3d`` calls it once per forward, the spatial GRU once per step."""
    if not (bn.training and bn.track_running_stats):
        return
    with torch.no_grad():
        factor = 0.0 if bn.momentum is None else bn.momentum
        if bn.num_batches_tracked is not None:
            bn.num_batches_tracked.add_(1)
            if bn.momentum is None and bn.running_mean is not None:
                factor = bn.num_batches_tracked.to(bn.running_mean.dtype).reciprocal()
        if bn.running_mean is None:
            return
        bn.running_mean.lerp_(mean.to(bn.running_mean.dtype), factor)
        bn.running_var.lerp_(var.to(bn.running_var.dtype) * (n / (n - 1)), factor)


def norm_act(norm: nn.Module, activation: nn.Module, y: torch.Tensor, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``activation(norm(y))``, plus ``residual`` when given (``residual + activation(norm(y))``): one fused apply when the norm is a
    ``FusedBatchNorm3d`` and the activation an ``nn.ReLU``, otherwise exactly those module calls and that add."""
    if isinstance(norm, FusedBatchNorm3d) and isinstance(activation, nn.ReLU):
        return norm.forward_act(y, relu=True, residual=residual)
    out = activation(norm(y))
    return out if residual is None else residual + out


from . import ops as _ops  # noqa: E402,F401  (registers torch.ops.fiery_b200.batch_norm_act)
