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

import math
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


def _workspace(d: _lib.BatchNormDesc, device: torch.device, group: bool = False) -> torch.Tensor:
    """The workspace of a call with ``d``; ``group``: of a rank in a group, whose batch may be 0."""
    lib = _lib.load()
    return _lib.workspace(lib.fiery_batch_norm_sync_workspace_bytes(d) if group else lib.fiery_batch_norm_workspace_bytes(d), device)


def _ptr(t: Optional[torch.Tensor]) -> int:
    """t's device address, 0 for None or an empty tensor (a rank with no values)."""
    return t.data_ptr() if t is not None and t.numel() else 0


def _forward_operands(x: torch.Tensor, weight, bias, residual):
    """(weight, bias, residual, y, mean, var) of a forward over x: the operands as the kernels read them, and the outputs."""
    c = int(x.shape[1])
    w, bs = _per_channel(weight, c, "weight"), _per_channel(bias, c, "bias")
    if residual is not None and tuple(residual.shape) != tuple(x.shape):
        raise ValueError(f"batch norm: residual {tuple(residual.shape)} does not match x {tuple(x.shape)}")
    r = f32(residual) if residual is not None else None
    y = torch.empty(tuple(x.shape), dtype=torch.float32, device=x.device)
    mean = torch.empty(c, dtype=torch.float32, device=x.device)
    var = torch.empty(c, dtype=torch.float32, device=x.device)
    return w, bs, r, y, mean, var


def _param_grads(c: int, device: torch.device, need_weight: bool, need_bias: bool):
    """(grad_weight, grad_bias): (C,) fp32 outputs, None where not asked for."""
    new = lambda: torch.empty(c, dtype=torch.float32, device=device)           # noqa: E731
    return new() if need_weight else None, new() if need_bias else None


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
    w, bs, r, y, mean, var = _forward_operands(xs, weight, bias, residual)
    rm, rv = _per_channel(running_mean, c, "running_mean"), _per_channel(running_var, c, "running_var")
    if not training and (rm is None or rv is None):
        raise ValueError("batch norm: eval mode needs running_mean and running_var")
    d = _desc(xs, training, relu, eps)
    _lib.call("fiery_batch_norm_forward", x.device, d, xs.data_ptr(), _ptr(w), _ptr(bs), _ptr(rm), _ptr(rv), _ptr(r), y.data_ptr(),
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
    dw, db = _param_grads(c, x.device, need_weight, need_bias)
    d = _desc(xs, training, relu, eps)
    _lib.call("fiery_batch_norm_backward", x.device, d, xs.data_ptr(), g.data_ptr(), _ptr(w), _ptr(bs), f32(mean).data_ptr(),
              f32(var).data_ptr(), _ptr(dx), _ptr(dw), _ptr(db), _workspace(d, x.device).data_ptr())
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


def update_running_stats(bn: nn.Module, mean: torch.Tensor, var: torch.Tensor, n) -> None:
    """``_BatchNorm.forward``'s bookkeeping on the norm ``bn`` for a batch of n values per channel with this mean and biased variance,
    as device tensor operations: nothing in eval or without tracked statistics, else ``num_batches_tracked += 1`` and each running
    statistic moved toward the batch's by the momentum (``1 / num_batches_tracked`` when the momentum is None), the variance as the
    unbiased n / (n - 1) var.  n is an int, or a one-element fp64 device tensor (a group's count, which the host never sees).
    ``FusedBatchNorm3d`` calls it once per forward, the spatial GRU once per step."""
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
        unbiased = (n / (n - 1)).to(bn.running_var.dtype) if isinstance(n, torch.Tensor) else n / (n - 1)
        bn.running_mean.lerp_(mean.to(bn.running_mean.dtype), factor)
        bn.running_var.lerp_(var.to(bn.running_var.dtype) * unbiased, factor)


# ------------------------------------------------------------------------------------------------------------------------------
# statistics over a process group (torch.nn.SyncBatchNorm): each rank's (C, 3) fp64 triplets are gathered, never all-reduced, and
# the kernels merge them in ascending rank order, so every rank gets bit-identical statistics
# ------------------------------------------------------------------------------------------------------------------------------
def gather(t: torch.Tensor, group) -> torch.Tensor:
    """(world, *t.shape): every rank's ``t`` in rank order, as torch's SyncBatchNorm gathers (``all_gather`` on gloo, else
    ``all_gather_into_tensor``)."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    if dist.get_backend(group) == "gloo":
        parts = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(parts, t, group)
        return torch.stack(parts)
    out = t.new_empty((world,) + tuple(t.shape))
    dist.all_gather_into_tensor(out, t, group)
    return out


def local_stats(x: torch.Tensor) -> torch.Tensor:
    """x (b, C, s, X, Y) fp32 with contiguous pixel planes (``f32_planes``), b may be 0 -> this rank's (C, 3) fp64 (n, mean, M2)."""
    d = _desc(x, True, False, 0.0)
    stats = torch.empty((x.shape[1], 3), dtype=torch.float64, device=x.device)
    _lib.call("fiery_batch_norm_local_stats", x.device, d, _ptr(x), stats.data_ptr(), _workspace(d, x.device, group=True).data_ptr())
    return stats


def _check_gathered(gathered: torch.Tensor, x: torch.Tensor) -> None:
    """The kernels read ``gathered`` as contiguous (world, C, 3) fp64 on x's device; anything else would be read as other numbers."""
    c = int(x.shape[1])
    if (gathered.dtype != torch.float64 or gathered.dim() != 3 or gathered.shape[0] < 1 or tuple(gathered.shape[1:]) != (c, 3)
            or not gathered.is_contiguous() or gathered.device != x.device):
        raise ValueError(f"batch norm: gathered must be a contiguous (world, {c}, 3) fp64 tensor, got {tuple(gathered.shape)} "
                         f"{gathered.dtype} with strides {gathered.stride()} on {gathered.device}")


def forward_gathered(gathered: torch.Tensor, x: torch.Tensor, weight, bias, residual, eps: float, relu: bool):
    """(y, mean, var, count) from the group's gathered (world, C, 3) triplets: y ``relu(batch_norm(x)) + residual`` with the group's
    mean and biased var, count the group's n as a (1,) fp64 device tensor."""
    _check_gathered(gathered, x)
    w, bs, r, y, mean, var = _forward_operands(x, weight, bias, residual)
    count = torch.empty(1, dtype=torch.float64, device=x.device)
    d = _desc(x, True, relu, eps)
    _lib.call("fiery_batch_norm_forward_gathered", x.device, d, int(gathered.shape[0]), gathered.data_ptr(), _ptr(x), _ptr(w), _ptr(bs),
              _ptr(r), _ptr(y), mean.data_ptr(), var.data_ptr(), count.data_ptr(), _workspace(d, x.device, group=True).data_ptr())
    return y, mean, var, count


def local_grad_sums(grad_y: torch.Tensor, x: torch.Tensor, weight, bias, mean, var, eps: float, relu: bool, need_weight: bool,
                    need_bias: bool):
    """(sums, grad_weight, grad_bias): this rank's (C, 3) fp64 (n, S1, S2) and its own weight and bias gradients (None where not
    asked for)."""
    c = int(x.shape[1])
    w, bs = _per_channel(weight, c, "weight"), _per_channel(bias, c, "bias")
    dw, db = _param_grads(c, x.device, need_weight, need_bias)
    sums = torch.empty((c, 3), dtype=torch.float64, device=x.device)
    d = _desc(x, True, relu, eps)
    _lib.call("fiery_batch_norm_local_grad_sums", x.device, d, _ptr(x), _ptr(grad_y), _ptr(w), _ptr(bs), mean.data_ptr(), var.data_ptr(),
              sums.data_ptr(), _ptr(dw), _ptr(db), _workspace(d, x.device, group=True).data_ptr())
    return sums, dw, db


def backward_gathered(gathered: torch.Tensor, grad_y: torch.Tensor, x: torch.Tensor, weight, bias, mean, var, eps: float,
                      relu: bool) -> torch.Tensor:
    """grad_x (contiguous fp32) from the group's gathered (world, C, 3) (n, S1, S2)."""
    c = int(x.shape[1])
    _check_gathered(gathered, x)
    w, bs = _per_channel(weight, c, "weight"), _per_channel(bias, c, "bias")
    dx = torch.empty(tuple(x.shape), dtype=torch.float32, device=x.device)
    d = _desc(x, True, relu, eps)
    _lib.call("fiery_batch_norm_backward_gathered", x.device, d, int(gathered.shape[0]), gathered.data_ptr(), _ptr(x), _ptr(grad_y), _ptr(w),
              _ptr(bs), mean.data_ptr(), var.data_ptr(), _ptr(dx), _workspace(d, x.device, group=True).data_ptr())
    return dx


class SyncBatchNormAct(torch.autograd.Function):
    """``relu(batch_norm(x)) + residual`` with a group's statistics: local stats, one ``gather``, apply; the backward local sums, one
    ``gather`` (when x needs its gradient), grad apply.  ``gather`` maps a (C, 3) fp64 tensor to the (world, C, 3) of every rank's,
    in rank order.  Returns (y, mean, var, count), the last three not differentiable."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, eps: float, relu: bool, gather):
        xs = f32_planes(x)
        gathered = gather(local_stats(xs))
        y, mean, var, count = forward_gathered(gathered, xs, weight, bias, residual, eps, relu)
        ctx.mark_non_differentiable(mean, var, count)
        ctx.eps, ctx.relu, ctx.gather = eps, relu, gather
        ctx.x_dtype = x.dtype
        ctx.residual_dtype = residual.dtype if residual is not None else None
        ctx.save_for_backward(xs, weight, bias, mean, var)
        return y, mean, var, count

    @staticmethod
    def backward(ctx, grad_y, _gm, _gv, _gc):
        xs, weight, bias, mean, var = ctx.saved_tensors
        need = ctx.needs_input_grad
        g = f32(grad_y)
        sums, dw, db = local_grad_sums(g, xs, weight, bias, mean, var, ctx.eps, ctx.relu, bool(need[1]), bool(need[2]))
        dx = None
        if need[0]:
            dx = backward_gathered(ctx.gather(sums), g, xs, weight, bias, mean, var, ctx.eps, ctx.relu).to(ctx.x_dtype)
        cast = lambda t, like: t.to(like.dtype) if t is not None else None           # noqa: E731
        grad_r = grad_y.to(ctx.residual_dtype) if need[3] else None
        return dx, cast(dw, weight), cast(db, bias), grad_r, None, None, None


def sync_group(norm: nn.Module):
    """The process group whose statistics ``norm`` (a SyncBatchNorm) uses in this call, or None when it uses its own batch's:
    torch's rule -- training with batch statistics, torch.distributed initialized, and a group of more than one rank."""
    import torch.distributed as dist
    batch_stats = norm.training or (norm.running_mean is None and norm.running_var is None)
    if not (batch_stats and norm.training and dist.is_available() and dist.is_initialized()):
        return None
    group = norm.process_group if norm.process_group is not None else dist.group.WORLD
    return group if dist.get_world_size(group) > 1 else None


class FusedSyncBatchNorm(nn.SyncBatchNorm):
    """Drop-in for an ``nn.SyncBatchNorm`` that runs on the batch-norm kernels.  It adopts the module's Parameters, buffers and
    ``process_group`` (the same objects: ``state_dict`` keys are unchanged).  When ``SyncBatchNorm`` would synchronize (training, batch
    statistics, torch.distributed initialized, a group of more than one rank) it runs ``SyncBatchNormAct``: every rank's (n, mean, M2)
    gathered and merged in rank order on the device, one gather forward and one backward, the running statistics moved with the
    group's count without a host synchronisation.  Otherwise it computes exactly what ``FusedBatchNorm3d`` does.  Inputs of any rank
    >= 2 are read as (b, C, 1, 1, rest) unless they are 5-D, and one with no elements as (0, C, 1, 1, 1): such a rank takes part in
    the gathers with n = 0, as in torch's SyncBatchNorm.  ``forward_act(x, relu, residual)`` is the fused entry."""

    def __init__(self, bn: nn.SyncBatchNorm):
        FusedBatchNorm3d.__init__(self, bn)
        self.process_group = bn.process_group

    forward = FusedBatchNorm3d.forward
    update_running_stats = FusedBatchNorm3d.update_running_stats

    def forward_act(self, x: torch.Tensor, relu: bool, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        self._check_input_dim(x)
        shape = x.shape
        if x.numel() == 0:                                # an empty rank, whichever dim is 0: batch 0 takes part with n = 0, where
            x = x.reshape(0, shape[1], 1, 1, 1)           # a plane of 0 pixels is not a valid shape
            residual = residual.reshape(x.shape) if residual is not None else None
        elif x.dim() != 5:
            x = x.reshape(shape[0], shape[1], 1, 1, math.prod(shape[2:]))
            residual = residual.reshape(x.shape) if residual is not None else None
        group = sync_group(self)
        if group is None:
            y = FusedBatchNorm3d.forward_act(self, x, relu, residual)
        else:
            _require_cuda(x, "x")
            y, mean, var, count = SyncBatchNormAct.apply(x, self.weight, self.bias, residual, self.eps, relu,
                                                           lambda t: gather(t, group))
            self.update_running_stats(mean, var, count)
        return y.reshape(shape)


def norm_act(norm: nn.Module, activation: nn.Module, y: torch.Tensor, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``activation(norm(y))``, plus ``residual`` when given (``residual + activation(norm(y))``): one fused apply when the norm is a
    ``FusedBatchNorm3d`` or a ``FusedSyncBatchNorm`` and the activation an ``nn.ReLU``, otherwise exactly those module calls and that
    add."""
    if isinstance(norm, (FusedBatchNorm3d, FusedSyncBatchNorm)) and isinstance(activation, nn.ReLU):
        return norm.forward_act(y, relu=True, residual=residual)
    out = activation(norm(y))
    return out if residual is None else residual + out


from . import ops as _ops  # noqa: E402,F401  (registers torch.ops.fiery_b200.batch_norm_act)
