"""The lift as dispatcher-visible operators: ``torch.ops.fiery_b200.lift_splat`` / ``lift_splat_backward``.

``torch.library.custom_op`` registrations on top of the same C ABI (libfiery_b200.so), so the fused lift is an operator the
dispatcher knows: it has a fake (meta) implementation for tracing / ``torch.compile``, an autograd formula registered with
``register_autograd`` (no Python ``autograd.Function`` in the graph), and an autocast rule that mirrors the reference -- under AMP
the reference's softmax and outer product run in fp32 (fiery/models/encoder.py:99-100 under autocast), so the operator's inputs are
cast to fp32.

One operator serves both lifts: the plain lift (``LiftSplat.forward``) and, given the warp's ``theta`` and ``copy_mask``, the lift with
``cumulative_warp_features`` in its layout pass (``LiftSplat.forward_warped``).  The operator also decides whether to make the
geometry plan that the forward and the backward share.

The operators take plain tensors plus an integer ``handle`` naming the ``LiftSplat`` module that holds the frustum / BEV-grid
constants (a registry of weak references; the constants are tiny host-derived tensors, not operator inputs).

The tensor-core layers' operators follow: ``temporal_entry`` here, and ``first_conv`` and ``causal_conv3d``, which their layer modules
(fiery_b200/bev_conv.py, fiery_b200/causal_conv.py) register through ``_register_conv``.  Importing this module registers them all.
"""
from __future__ import annotations

import weakref
from typing import List, Optional, Tuple

import torch

from .lift import _plan_bytes
from .warp import _warp_adjoint

_REGISTRY = {}          # handle -> (weakref to the LiftSplat module, (C, X, Y, feat_w, channels_last) as python values for the fakes)


def register_module(module, device: torch.device) -> int:
    handle = id(module)
    c = module._constants(device)                                    # cached host-side integers: no device sync here
    X, Y, _ = c["dim"]
    meta = (int(module.encoder_out_channels), int(X), int(Y), int(c["w"]), module.output_layout == "channels_last")
    entry = _REGISTRY.get(handle)
    if entry is None or entry[0]() is not module or entry[1] != meta:
        _REGISTRY[handle] = (weakref.ref(module, lambda _r, h=handle: _REGISTRY.pop(h, None)), meta)
    return handle


def _module(handle: int):
    entry = _REGISTRY.get(handle)
    m = entry[0]() if entry is not None else None
    if m is None:
        raise RuntimeError("fiery_b200::lift_splat: the LiftSplat module behind this handle is gone")
    return m


@torch.library.custom_op("fiery_b200::lift_splat", mutates_args=(), device_types="cuda")
def lift_splat(head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor, plan: Optional[torch.Tensor], handle: int,
               make_plan: bool, theta: Optional[torch.Tensor] = None,
               copy_mask: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(head (B'n, D+C, h, w), intrinsics (B', n, 3, 3), extrinsics (B', n, 4, 4)) -> (BEV (B', C, X, Y) fp32, plan).
    ``plan``: a geometry plan of this calibration, or None.  ``make_plan``: compute one (returned, for the backward) when none was
    passed; otherwise the second output is an empty tensor and the tile kernels evaluate the geometry themselves.
    ``theta`` (B', 2, 3) fp32 and ``copy_mask`` (B',) uint8: the warped lift -- every frame is sampled under its map in the layout
    pass (fiery_lift_forward_warped) and the BEV is NCHW whatever the module's output layout."""
    m = _module(handle)
    made = None
    if plan is None and make_plan and intrinsics.shape[0]:
        made = m.plan(intrinsics.to(head.device), extrinsics)
    out = m._launch_forward(head, intrinsics, extrinsics, plan=plan if plan is not None else made,
                            warp=(theta, copy_mask) if theta is not None else None)
    # the second output is the plan MADE here (an operator output may not alias an input: a plan that was passed in is not returned)
    return out, (made if made is not None else torch.empty(0, dtype=torch.uint8, device=head.device))


@lift_splat.register_fake
def _(head, intrinsics, extrinsics, plan, handle, make_plan, theta=None, copy_mask=None):
    # python values only: nothing here touches a real tensor.  Under dynamic shapes the handle may arrive as a SymInt: int()
    # specialises the graph on it (it names one module)
    C, X, Y, feat_w, channels_last = _REGISTRY[int(handle)][1]
    B, n = intrinsics.shape[:2]
    bev = head.new_empty((B, X, Y, C), dtype=torch.float32).permute(0, 3, 1, 2) if channels_last and theta is None \
        else head.new_empty((B, C, X, Y), dtype=torch.float32)
    # the plan made here (fiery_lift_plan_bytes bytes; 0 for B' = 0, where the real op makes none), else an empty tensor
    plan_bytes = _plan_bytes(B, n, feat_w, X * Y) if plan is None and make_plan else 0
    return bev, head.new_empty((plan_bytes,), dtype=torch.uint8)


@torch.library.custom_op("fiery_b200::lift_splat_backward", mutates_args=(), device_types="cuda")
def lift_splat_backward(head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor, grad_bev: torch.Tensor,
                        plan: Optional[torch.Tensor], handle: int, theta: Optional[torch.Tensor] = None,
                        copy_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Gradient of the BEV w.r.t. the head tensor (same shape and dtype as ``head``); the calibration gets none (geometry.py:300).
    With ``theta`` / ``copy_mask`` (the warped lift) ``grad_bev`` first goes through the warp's adjoint.  Both steps run inside this
    operator, so the backward graph holds dispatcher operators only.  Folding the adjoint into the gradient's re-layout pass was
    built and measured slower, so the two launches stay separate."""
    if theta is not None:
        grad_bev = _warp_adjoint(grad_bev, theta, copy_mask, 0)      # the warped lift samples bilinearly
    return _module(handle)._launch_backward(head, intrinsics, extrinsics, grad_bev,
                                            plan=plan if (plan is not None and plan.numel()) else None)


@lift_splat_backward.register_fake
def _(head, intrinsics, extrinsics, grad_bev, plan, handle, theta=None, copy_mask=None):
    return head.new_empty(head.shape)                                # NCHW-contiguous whatever the head's layout, like the op


def _setup_context(ctx, inputs, output):
    head, intrinsics, extrinsics, plan, handle, _make_plan, theta, copy_mask = inputs
    _bev, plan_out = output
    ctx.handle = handle
    ctx.save_for_backward(head, intrinsics, extrinsics, plan if plan is not None else plan_out, theta, copy_mask)


def _backward(ctx, grad_bev, _grad_plan):
    head, intrinsics, extrinsics, plan, theta, copy_mask = ctx.saved_tensors
    grad_head = torch.ops.fiery_b200.lift_splat_backward(head, intrinsics, extrinsics, grad_bev, plan, ctx.handle, theta, copy_mask)
    return grad_head, None, None, None, None, None, None, None


lift_splat.register_autograd(_backward, setup_context=_setup_context)
# AMP (baseline.yml PRECISION 16): the reference's softmax / outer product run in fp32 under autocast -> so does the operator
torch.library.register_autocast("fiery_b200::lift_splat", "cuda", torch.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# Convolutions of one input by one weight as dispatcher operators ``fiery_b200::<name>`` / ``<name>_backward``, each registered by
# its layer module with the forward, the two gradients and the fake shapes: ``first_conv`` (Decoder.first_conv,
# fiery/models/decoder.py:11,59; fiery_b200/bev_conv.py) and ``causal_conv3d`` (CausalConv3d's pad + Conv3d,
# fiery/layers/temporal.py:65-85; fiery_b200/causal_conv.py).
# Autocast: the operators run in fp32 (TF32 tensor-core operands, fp32 accumulation) -- under AMP the reference runs these
# convolutions in fp16, so an AMP step computes them at a higher precision than the reference does.
# ------------------------------------------------------------------------------------------------------------------------------
def _cast_back(grad: Optional[torch.Tensor], like: torch.Tensor) -> torch.Tensor:
    """``grad`` in the dtype of the tensor it is the gradient of; a gradient that was not asked for (None) comes back as an empty
    tensor (an operator returns tensors)."""
    if grad is None:
        return like.new_empty((0,))
    return grad if grad.dtype == like.dtype else grad.to(like.dtype)


def _register_conv(name: str, forward, grad_layout, grad_input, grad_weight, fake_output, fake_grad_input) -> None:
    """``fiery_b200::<name>(x, weight) = forward(x, weight)`` and ``<name>_backward(grad_y, x, weight, need_input, need_weight)
    -> (grad_x, grad_weight)``: grad_y is converted once by ``grad_layout`` and shared by ``grad_input(g, x, weight)`` and
    ``grad_weight(g, x, weight)``; only the gradients asked for are computed, in x's and the weight's dtype.  The fakes take their
    shapes and strides from ``fake_output(x, weight)`` and ``fake_grad_input(x)``; the weight gradient has the weight's shape."""
    @torch.library.custom_op(f"fiery_b200::{name}", mutates_args=(), device_types="cuda")
    def op(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
        return forward(x, weight)

    op.register_fake(fake_output)

    @torch.library.custom_op(f"fiery_b200::{name}_backward", mutates_args=(), device_types="cuda")
    def backward_op(grad_y: torch.Tensor, x: torch.Tensor, weight: torch.Tensor, need_input: bool,
                    need_weight: bool) -> Tuple[torch.Tensor, torch.Tensor]:
        g = grad_layout(grad_y)
        return (_cast_back(grad_input(g, x, weight) if need_input else None, x),
                _cast_back(grad_weight(g, x, weight) if need_weight else None, weight))

    @backward_op.register_fake
    def _(grad_y, x, weight, need_input, need_weight):
        return (fake_grad_input(x) if need_input else x.new_empty((0,)),
                weight.new_empty(weight.shape) if need_weight else weight.new_empty((0,)))

    def setup_context(ctx, inputs, output):
        ctx.save_for_backward(*inputs)

    def backward(ctx, grad_y):
        x, weight = ctx.saved_tensors
        need_input, need_weight = bool(ctx.needs_input_grad[0]), bool(ctx.needs_input_grad[1])
        if not (need_input or need_weight):
            return None, None
        grad_x, grad_w = backward_op(grad_y, x, weight, need_input, need_weight)
        return (grad_x if need_input else None), (grad_w if need_weight else None)

    op.register_autograd(backward, setup_context=setup_context)
    torch.library.register_autocast(f"fiery_b200::{name}", "cuda", torch.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# The temporal block's 1x1x1 input projections (TemporalBlock, fiery/layers/temporal.py:218-281) as dispatcher operators:
# ``torch.ops.fiery_b200.temporal_entry`` / ``temporal_entry_backward`` (fiery_b200/temporal.py; kernels in csrc/temporal_entry.cu).
# Autocast: the operator runs in fp32 (TF32 tensor-core operands, fp32 accumulation), as first_conv does; under AMP the reference runs
# these convolutions in fp16.
# ------------------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op("fiery_b200::temporal_entry", mutates_args=(), device_types="cuda")
def temporal_entry(x: torch.Tensor, weights: List[torch.Tensor], extra: Optional[torch.Tensor]) -> List[torch.Tensor]:
    """x (b, K, s, X, Y), any strides; weights: 1..4 Conv3d weights (C_q, K + E, 1, 1, 1); extra (b, s, E) per-frame channels that
    are constant over the map (E = 0: None).  Returns one contiguous (b, C_q, s, X, Y) fp32 tensor per weight: the 1x1x1 convolution
    of ``cat([x, extra broadcast over the map], 1)``.  The weights' pack is made at most once per weight version."""
    from .temporal import entry_forward
    return entry_forward(x, weights, extra)


@temporal_entry.register_fake
def _(x, weights, extra):
    b, _, s, h, w = x.shape
    return [x.new_empty((b, wt.shape[0], s, h, w), dtype=torch.float32) for wt in weights]


@torch.library.custom_op("fiery_b200::temporal_entry_backward", mutates_args=(), device_types="cuda")
def temporal_entry_backward(grads: List[torch.Tensor], x: torch.Tensor, weights: List[torch.Tensor], extra: Optional[torch.Tensor],
                            need_input: bool, need_weight: bool) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """(grad_x, grad_weights) of ``temporal_entry``; a gradient that is not asked for is not computed and comes back empty.
    grad_x: x's shape and dtype, with x's strides where the kernels read x as it lies (``temporal.input_strides``); grad_weights: each
    weight's shape and dtype, bit-reproducible (no atomics).  extra gets no gradient."""
    from .temporal import entry_backward_data, entry_backward_weight
    grad_x = _cast_back(entry_backward_data(grads, x, weights) if need_input else None, x)
    grad_w = entry_backward_weight(grads, x, weights, extra) if need_weight else [None] * len(weights)
    return grad_x, [_cast_back(g, wt) for g, wt in zip(grad_w, weights)]


@temporal_entry_backward.register_fake
def _(grads, x, weights, extra, need_input, need_weight):
    from .temporal import input_strides
    grad_x = x.new_empty_strided(tuple(x.shape), input_strides(tuple(x.shape), x.stride())) if need_input else x.new_empty((0,))
    grad_w = [wt.new_empty(wt.shape) if need_weight else wt.new_empty((0,)) for wt in weights]
    return grad_x, grad_w


def _temporal_entry_setup_context(ctx, inputs, output):
    x, weights, extra = inputs
    ctx.n_weights = len(weights)
    ctx.save_for_backward(x, extra, *weights)


def _temporal_entry_backward(ctx, grads):
    x, extra, *weights = ctx.saved_tensors
    # a tensor-list input's needs_input_grad is a list, and its gradient must be a list of the same length
    need_input, need_w = bool(ctx.needs_input_grad[0]), [bool(n) for n in ctx.needs_input_grad[1]]
    if not (need_input or any(need_w)):
        return None, [None] * len(weights), None
    grads = [g if g is not None else torch.zeros((x.shape[0], wt.shape[0], *x.shape[2:]), dtype=torch.float32, device=x.device)
             for g, wt in zip(grads, weights)]
    grad_x, grad_w = torch.ops.fiery_b200.temporal_entry_backward(grads, x, weights, extra, need_input, any(need_w))
    return (grad_x if need_input else None), [g if n else None for g, n in zip(grad_w, need_w)], None


temporal_entry.register_autograd(_temporal_entry_backward, setup_context=_temporal_entry_setup_context)
torch.library.register_autocast("fiery_b200::temporal_entry", "cuda", torch.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# The temporal block's pyramid pooling and aggregation (fiery/layers/temporal.py:167-215, 268-276): ``spatial_sums`` (the pooling's
# spatial means; csrc/spatial_sums.cu) and ``temporal_aggregation`` (the aggregation conv of the paths and the broadcast pooled vector,
# without the concat or the broadcast; the entry's kernels in swapped roles).  Autocast: both run in fp32.
# ------------------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op("fiery_b200::spatial_sums", mutates_args=(), device_types="cuda")
def spatial_sums(x: torch.Tensor) -> torch.Tensor:
    """x (b, C, s, X, Y) -> (b, C, s) fp32 sums over each pixel plane; the order depends on X*Y only (bit-identical for a plane
    whatever its strides or neighbours).  Its gradient is the broadcast of the output gradient over the map."""
    from .temporal import spatial_sums as sums
    return sums(x)


@spatial_sums.register_fake
def _(x):
    return x.new_empty(tuple(x.shape[:3]), dtype=torch.float32)


def _spatial_sums_setup_context(ctx, inputs, output):
    (x,) = inputs
    ctx.x_shape, ctx.x_dtype = tuple(x.shape), x.dtype


def _spatial_sums_backward(ctx, grad):
    return grad[..., None, None].to(ctx.x_dtype).expand(ctx.x_shape)


spatial_sums.register_autograd(_spatial_sums_backward, setup_context=_spatial_sums_setup_context)
torch.library.register_autocast("fiery_b200::spatial_sums", "cuda", torch.float32)


@torch.library.custom_op("fiery_b200::temporal_aggregation", mutates_args=(), device_types="cuda")
def temporal_aggregation(paths: List[torch.Tensor], weight: torch.Tensor, pooled: torch.Tensor) -> torch.Tensor:
    """paths: 1..4 tensors (b, C_q, s, X, Y); weight (N, sum C_q + R, 1, 1, 1), the aggregation's bias-free 1x1x1 Conv3d; pooled
    (b, R, s), constant over the map.  Returns the contiguous (b, N, s, X, Y) fp32 ``conv3d(cat([*paths, pooled broadcast], 1),
    weight)`` without building the concat or the broadcast.  The weight's pack is made at most once per weight version."""
    from .temporal import aggregation_forward
    return aggregation_forward(paths, weight, pooled)


@temporal_aggregation.register_fake
def _(paths, weight, pooled):
    b, _, s, h, w = paths[0].shape
    return paths[0].new_empty((b, weight.shape[0], s, h, w), dtype=torch.float32)


@torch.library.custom_op("fiery_b200::temporal_aggregation_backward", mutates_args=(), device_types="cuda")
def temporal_aggregation_backward(grad: torch.Tensor, paths: List[torch.Tensor], weight: torch.Tensor, pooled: torch.Tensor,
                                  need_paths: bool, need_weight: bool,
                                  need_pooled: bool) -> Tuple[List[torch.Tensor], torch.Tensor, torch.Tensor]:
    """(grad_paths, grad_weight, grad_pooled) of ``temporal_aggregation``, each in its input's shape and dtype (the paths' gradients
    contiguous); a gradient that is not asked for is not computed and comes back empty.  The weight gradient is bit-reproducible."""
    from .temporal import aggregation_backward
    gp, gw, gv = aggregation_backward(grad, paths, weight, pooled, need_paths, need_weight, need_pooled)
    return ([_cast_back(g, p) for g, p in zip(gp, paths)] if gp is not None else [p.new_empty((0,)) for p in paths],
            _cast_back(gw, weight), _cast_back(gv, pooled))


@temporal_aggregation_backward.register_fake
def _(grad, paths, weight, pooled, need_paths, need_weight, need_pooled):
    return ([p.new_empty(p.shape) if need_paths else p.new_empty((0,)) for p in paths],
            weight.new_empty(weight.shape) if need_weight else weight.new_empty((0,)),
            pooled.new_empty(pooled.shape) if need_pooled else pooled.new_empty((0,)))


def _temporal_aggregation_setup_context(ctx, inputs, output):
    paths, weight, pooled = inputs
    ctx.save_for_backward(weight, pooled, *paths)


def _temporal_aggregation_backward(ctx, grad):
    weight, pooled, *paths = ctx.saved_tensors
    need_p, need_w, need_v = any(bool(n) for n in ctx.needs_input_grad[0]), bool(ctx.needs_input_grad[1]), bool(ctx.needs_input_grad[2])
    if not (need_p or need_w or need_v):
        return [None] * len(paths), None, None
    gp, gw, gv = torch.ops.fiery_b200.temporal_aggregation_backward(grad, paths, weight, pooled, need_p, need_w, need_v)
    return ([g if n else None for g, n in zip(gp, ctx.needs_input_grad[0])], gw if need_w else None, gv if need_v else None)


temporal_aggregation.register_autograd(_temporal_aggregation_backward, setup_context=_temporal_aggregation_setup_context)
torch.library.register_autocast("fiery_b200::temporal_aggregation", "cuda", torch.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# The temporal model's BatchNorm3d with its ReLU and the block's residual add (fiery/layers/temporal.py:107-117, 65-85, 256-281):
# ``batch_norm_act`` / ``batch_norm_act_backward`` (fiery_b200/batch_norm.py; kernels in csrc/batch_norm.cu).  The statistics
# outputs are not differentiable and the operator updates no running buffer (FusedBatchNorm3d does, from them).  Autocast: fp32,
# like the other temporal operators; a 16-bit input is widened and the output is fp32.
# ------------------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op("fiery_b200::batch_norm_act", mutates_args=(), device_types="cuda")
def batch_norm_act(x: torch.Tensor, weight: Optional[torch.Tensor], bias: Optional[torch.Tensor], running_mean: Optional[torch.Tensor],
                   running_var: Optional[torch.Tensor], residual: Optional[torch.Tensor], training: bool, eps: float,
                   relu: bool) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """x (b, C, s, X, Y), pixel planes read as they lie -> (y, mean, var): y the contiguous fp32 ``relu(batch_norm(x)) + residual``
    (the ReLU when ``relu``, the add when ``residual`` is given), mean and the biased var the (C,) fp32 statistics used: the batch's
    when ``training``, else copies of ``running_mean`` / ``running_var``.  Bit-reproducible: the order depends on the shape only."""
    from .batch_norm import forward
    return forward(x, weight, bias, running_mean, running_var, residual, training, eps, relu)


@batch_norm_act.register_fake
def _(x, weight, bias, running_mean, running_var, residual, training, eps, relu):
    c = x.shape[1]
    return (x.new_empty(tuple(x.shape), dtype=torch.float32), x.new_empty((c,), dtype=torch.float32),
            x.new_empty((c,), dtype=torch.float32))


@torch.library.custom_op("fiery_b200::batch_norm_act_backward", mutates_args=(), device_types="cuda")
def batch_norm_act_backward(grad_y: torch.Tensor, x: torch.Tensor, weight: Optional[torch.Tensor], bias: Optional[torch.Tensor],
                            mean: torch.Tensor, var: torch.Tensor, training: bool, eps: float, relu: bool, need_input: bool,
                            need_weight: bool, need_bias: bool) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(grad_x, grad_weight, grad_bias) of ``batch_norm_act``, each in its input's dtype (grad_x contiguous); a gradient that is not
    asked for is not computed and comes back empty.  Needs only x and the forward's (mean, var): the output is not kept."""
    from .batch_norm import backward
    dx, dw, db = backward(grad_y, x, weight, bias, mean, var, training, eps, relu, need_input, need_weight, need_bias)
    return _cast_back(dx, x), _cast_back(dw, weight if weight is not None else x), _cast_back(db, bias if bias is not None else x)


@batch_norm_act_backward.register_fake
def _(grad_y, x, weight, bias, mean, var, training, eps, relu, need_input, need_weight, need_bias):
    c = x.shape[1]
    return (x.new_empty(tuple(x.shape)) if need_input else x.new_empty((0,)),
            weight.new_empty((c,)) if need_weight else x.new_empty((0,)),
            bias.new_empty((c,)) if need_bias else x.new_empty((0,)))


def _batch_norm_act_setup_context(ctx, inputs, output):
    x, weight, bias, _rm, _rv, residual, training, eps, relu = inputs
    _y, mean, var = output
    ctx.mark_non_differentiable(mean, var)
    ctx.training, ctx.eps, ctx.relu = training, eps, relu
    ctx.residual_dtype = residual.dtype if residual is not None else None
    ctx.save_for_backward(x, weight, bias, mean, var)


def _batch_norm_act_backward(ctx, grad_y, _grad_mean, _grad_var):
    x, weight, bias, mean, var = ctx.saved_tensors
    need = ctx.needs_input_grad
    need_x, need_w, need_b, need_r = bool(need[0]), bool(need[1]), bool(need[2]), bool(need[5])
    dx = dw = db = None
    if need_x or need_w or need_b:
        dx, dw, db = torch.ops.fiery_b200.batch_norm_act_backward(grad_y, x, weight, bias, mean, var, ctx.training, ctx.eps, ctx.relu,
                                                                  need_x, need_w, need_b)
    grad_r = grad_y.to(ctx.residual_dtype) if need_r else None        # the residual is added as it is: its gradient is grad_y
    return (dx if need_x else None, dw if need_w else None, db if need_b else None, None, None, grad_r, None, None, None)


batch_norm_act.register_autograd(_batch_norm_act_backward, setup_context=_batch_norm_act_setup_context)
torch.library.register_autocast("fiery_b200::batch_norm_act", "cuda", torch.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# The future prediction's SpatialGRU (fiery/layers/temporal.py:10-62): ``spatial_gru`` / ``spatial_gru_backward``
# (fiery_b200/future_prediction.py; kernels in csrc/spatial_gru.cu).  The statistics and the saved tensors are not differentiable and
# the operator updates no running buffer (TensorCoreSpatialGRU does, from the statistics).  Autocast: fp32, like the temporal
# operators; under AMP the reference runs these convolutions in fp16.
# ------------------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op("fiery_b200::spatial_gru", mutates_args=(), device_types="cuda")
def spatial_gru(x: torch.Tensor, h0: torch.Tensor, w_update: torch.Tensor, b_update: torch.Tensor, w_reset: torch.Tensor,
                b_reset: torch.Tensor, w_state: torch.Tensor, bn_weight: Optional[torch.Tensor], bn_bias: Optional[torch.Tensor],
                running_mean: Optional[torch.Tensor], running_var: Optional[torch.Tensor], frames: int, training: bool, eps: float,
                bias_init: float) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """x (b, Tx, C_x, H, W) with Tx 1 (the same frame at every step) or ``frames``; h0 (b, C_h, H, W); the gates' (C_h, C_x + C_h, 3, 3)
    weights and (C_h,) biases, the state conv's bias-free weight, its BatchNorm2d's affine parameters (or None) and, in eval, its
    running statistics.  Returns (out, means, vars, saved): the contiguous (b, frames, C_h, H, W) fp32 states, the (frames, C_h)
    statistics each step normalized with, and a uint8 buffer the backward reads.  Bit-reproducible."""
    from .future_prediction import forward
    return forward(x, h0, w_update, b_update, w_reset, b_reset, w_state, bn_weight, bn_bias, running_mean, running_var, frames, training,
                   eps, bias_init)


@spatial_gru.register_fake
def _(x, h0, w_update, b_update, w_reset, b_reset, w_state, bn_weight, bn_bias, running_mean, running_var, frames, training, eps,
      bias_init):
    b, _, _, h, w = x.shape
    ch = w_update.shape[0]
    return (x.new_empty((b, frames, ch, h, w), dtype=torch.float32), x.new_empty((frames, ch), dtype=torch.float32),
            x.new_empty((frames, ch), dtype=torch.float32), x.new_empty((16 * frames * b * ch * h * w,), dtype=torch.uint8))


@torch.library.custom_op("fiery_b200::spatial_gru_backward", mutates_args=(), device_types="cuda")
def spatial_gru_backward(grad_out: torch.Tensor, x: torch.Tensor, h0: torch.Tensor, out: torch.Tensor, saved: torch.Tensor,
                         means: torch.Tensor, var: torch.Tensor, w_update: torch.Tensor, w_reset: torch.Tensor, w_state: torch.Tensor,
                         bn_weight: Optional[torch.Tensor], bn_bias: Optional[torch.Tensor], frames: int, training: bool, eps: float,
                         bias_init: float, need_x: bool, need_h0: bool, need_gates: bool, need_state: bool,
                         need_bn: bool) -> List[torch.Tensor]:
    """[grad_x, grad_h0, grad_w_update, grad_b_update, grad_w_reset, grad_b_reset, grad_w_state, grad_bn_weight, grad_bn_bias] of
    ``spatial_gru``, each in its input's shape and dtype; a gradient that is not asked for is not computed and comes back empty.  The
    recurrence runs in reverse; the weight gradients are bit-reproducible."""
    from .future_prediction import backward
    g = backward(grad_out, x, h0, out, saved, means, var, w_update, w_reset, w_state, bn_weight, bn_bias, frames, training, eps,
                 bias_init, need_x, need_h0, need_gates, need_state, need_bn)
    likes = (x, h0, w_update, w_update, w_reset, w_reset, w_state, bn_weight if bn_weight is not None else x,
             bn_bias if bn_bias is not None else x)
    return [_cast_back(gi, like) for gi, like in zip(g, likes)]


@spatial_gru_backward.register_fake
def _(grad_out, x, h0, out, saved, means, var, w_update, w_reset, w_state, bn_weight, bn_bias, frames, training, eps, bias_init,
      need_x, need_h0, need_gates, need_state, need_bn):
    ch = w_update.shape[0]
    e = x.new_empty((0,))
    return [x.new_empty(x.shape) if need_x else e, h0.new_empty(h0.shape) if need_h0 else e,
            w_update.new_empty(w_update.shape) if need_gates else e, w_update.new_empty((ch,)) if need_gates else e,
            w_reset.new_empty(w_reset.shape) if need_gates else e, w_reset.new_empty((ch,)) if need_gates else e,
            w_state.new_empty(w_state.shape) if need_state else e,
            bn_weight.new_empty((ch,)) if need_bn and bn_weight is not None else e,
            bn_bias.new_empty((ch,)) if need_bn and bn_bias is not None else e]


def _spatial_gru_setup_context(ctx, inputs, output):
    (x, h0, w_u, _b_u, w_r, _b_r, w_s, bn_w, bn_b, _rm, _rv, frames, training, eps, bias_init) = inputs
    out, means, var, saved = output
    ctx.mark_non_differentiable(means, var, saved)
    ctx.args = (frames, training, eps, bias_init)
    ctx.save_for_backward(x, h0, out, saved, means, var, w_u, w_r, w_s, bn_w, bn_b)


def _spatial_gru_backward(ctx, grad_out, _gm, _gv, _gs):
    x, h0, out, saved, means, var, w_u, w_r, w_s, bn_w, bn_b = ctx.saved_tensors
    n = ctx.needs_input_grad
    need_x, need_h0 = bool(n[0]), bool(n[1])
    need_gates, need_state, need_bn = bool(n[2] or n[3] or n[4] or n[5]), bool(n[6]), bool(n[7] or n[8])
    if not (need_x or need_h0 or need_gates or need_state or need_bn):
        return (None,) * 15
    if grad_out is None:
        grad_out = torch.zeros_like(out)
    g = torch.ops.fiery_b200.spatial_gru_backward(grad_out, x, h0, out, saved, means, var, w_u, w_r, w_s, bn_w, bn_b, *ctx.args,
                                                  need_x, need_h0, need_gates, need_state, need_bn)
    return tuple(gi if bool(ni) else None for gi, ni in zip(g, n[:9])) + (None,) * 6


spatial_gru.register_autograd(_spatial_gru_backward, setup_context=_spatial_gru_setup_context)
torch.library.register_autocast("fiery_b200::spatial_gru", "cuda", torch.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# The future prediction's Bottleneck (fiery/layers/convolutions.py:64-168, the plain variant): ``bottleneck`` / ``bottleneck_backward``
# (fiery_b200/bottleneck.py; csrc/bottleneck.cu).  Besides the output it returns the pre-norm maps y1, y2, y3 and the norms'
# statistics, which the backward reads; they are not differentiable, and the operator updates no running buffer
# (TensorCoreBottleneck does, from the statistics).  Autocast: fp32, like the other future-prediction operators.
# ------------------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op("fiery_b200::bottleneck", mutates_args=(), device_types="cuda")
def bottleneck(x: torch.Tensor, w_down: torch.Tensor, w_conv: torch.Tensor, w_up: torch.Tensor, bn1_weight: Optional[torch.Tensor],
               bn1_bias: Optional[torch.Tensor], bn1_mean: Optional[torch.Tensor], bn1_var: Optional[torch.Tensor],
               bn2_weight: Optional[torch.Tensor], bn2_bias: Optional[torch.Tensor], bn2_mean: Optional[torch.Tensor],
               bn2_var: Optional[torch.Tensor], bn3_weight: Optional[torch.Tensor], bn3_bias: Optional[torch.Tensor],
               bn3_mean: Optional[torch.Tensor], bn3_var: Optional[torch.Tensor], training: bool,
               eps: float) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """x (N, C, H, W) -> (out, y1, y2, y3, stats): out = relu(bn3(W_up relu(bn2(conv3x3(relu(bn1(W_down x))))))) + x, contiguous
    fp32; y1, y2 (N, C / 2, H, W) and y3 (N, C, H, W) the pre-norm maps; stats the (2 (2 (C / 2) + C),) fp32 means and biased
    variances each norm used (the batch's when ``training``, else copies of the running ones: bnI_mean / bnI_var).  Bit-reproducible."""
    from .bottleneck import forward
    return forward(x, w_down, w_conv, w_up, [bn1_weight, bn1_bias, bn1_mean, bn1_var, bn2_weight, bn2_bias, bn2_mean, bn2_var,
                                             bn3_weight, bn3_bias, bn3_mean, bn3_var], training, eps)


@bottleneck.register_fake
def _(x, w_down, w_conv, w_up, bn1_weight, bn1_bias, bn1_mean, bn1_var, bn2_weight, bn2_bias, bn2_mean, bn2_var, bn3_weight, bn3_bias,
      bn3_mean, bn3_var, training, eps):
    n, c, h, w = x.shape
    m = c // 2
    new = lambda *shape: x.new_empty(shape, dtype=torch.float32)  # noqa: E731
    return new(n, c, h, w), new(n, m, h, w), new(n, m, h, w), new(n, c, h, w), new(4 * m + 2 * c)


@torch.library.custom_op("fiery_b200::bottleneck_backward", mutates_args=(), device_types="cuda")
def bottleneck_backward(grad_out: torch.Tensor, x: torch.Tensor, y1: torch.Tensor, y2: torch.Tensor, y3: torch.Tensor,
                        stats: torch.Tensor, w_down: torch.Tensor, w_conv: torch.Tensor, w_up: torch.Tensor,
                        bn1_weight: Optional[torch.Tensor], bn1_bias: Optional[torch.Tensor], bn2_weight: Optional[torch.Tensor],
                        bn2_bias: Optional[torch.Tensor], bn3_weight: Optional[torch.Tensor], bn3_bias: Optional[torch.Tensor],
                        training: bool, eps: float, need: List[bool]) -> List[torch.Tensor]:
    """[grad_x, grad_w_down, grad_w_conv, grad_w_up, then each norm's grad weight and grad bias] of ``bottleneck``, each in its
    input's shape and dtype; ``need`` (10 flags in that order) says which are computed, the others come back empty."""
    from .bottleneck import backward
    norms = [bn1_weight, bn1_bias, None, None, bn2_weight, bn2_bias, None, None, bn3_weight, bn3_bias, None, None]
    g = backward(grad_out, x, y1, y2, y3, stats, w_down, w_conv, w_up, norms, training, eps, need)
    likes = [x, w_down, w_conv, w_up, bn1_weight, bn1_bias, bn2_weight, bn2_bias, bn3_weight, bn3_bias]
    return [_cast_back(gi, like if like is not None else x) for gi, like in zip(g, likes)]


@bottleneck_backward.register_fake
def _(grad_out, x, y1, y2, y3, stats, w_down, w_conv, w_up, bn1_weight, bn1_bias, bn2_weight, bn2_bias, bn3_weight, bn3_bias, training,
      eps, need):
    likes = [x, w_down, w_conv, w_up, bn1_weight, bn1_bias, bn2_weight, bn2_bias, bn3_weight, bn3_bias]
    return [like.new_empty(like.shape) if nd and like is not None else x.new_empty((0,)) for like, nd in zip(likes, need)]


def _bottleneck_setup_context(ctx, inputs, output):
    x, w_d, w_c, w_u, n1w, n1b, _m1, _v1, n2w, n2b, _m2, _v2, n3w, n3b, _m3, _v3, training, eps = inputs
    _out, y1, y2, y3, stats = output
    ctx.mark_non_differentiable(y1, y2, y3, stats)
    ctx.args = (training, eps)
    ctx.save_for_backward(x, y1, y2, y3, stats, w_d, w_c, w_u, n1w, n1b, n2w, n2b, n3w, n3b)


_BOTTLENECK_GRAD_SLOTS = (0, 1, 2, 3, 4, 5, 8, 9, 12, 13)          # the inputs bottleneck_backward's gradients belong to


def _bottleneck_backward(ctx, grad_out, _g1, _g2, _g3, _gs):
    x, y1, y2, y3, stats, w_d, w_c, w_u, n1w, n1b, n2w, n2b, n3w, n3b = ctx.saved_tensors
    need = [bool(ctx.needs_input_grad[i]) for i in _BOTTLENECK_GRAD_SLOTS]
    grads = [None] * 18
    if not any(need) or grad_out is None:
        return tuple(grads)
    g = torch.ops.fiery_b200.bottleneck_backward(grad_out, x, y1, y2, y3, stats, w_d, w_c, w_u, n1w, n1b, n2w, n2b, n3w, n3b, *ctx.args,
                                                 need)
    for slot, gi, nd in zip(_BOTTLENECK_GRAD_SLOTS, g, need):
        grads[slot] = gi if nd else None
    return tuple(grads)


bottleneck.register_autograd(_bottleneck_backward, setup_context=_bottleneck_setup_context)
torch.library.register_autocast("fiery_b200::bottleneck", "cuda", torch.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# The decoder's output heads after their 3x3 convolution (fiery/models/decoder.py:24-50): ``output_head`` / ``output_head_backward``
# (fiery_b200/decoder.py; csrc/output_head.cu).  The statistics outputs are not differentiable and the operator updates no running
# buffer (FusedOutputHead does, from them).  Autocast: fp32, like the other operators; a 16-bit y is widened once by the autocast cast
# and the gradients come back in the inputs' dtypes.
# ------------------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op("fiery_b200::output_head", mutates_args=(), device_types="cuda")
def output_head(y: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, bn_weight: Optional[torch.Tensor], bn_bias: Optional[torch.Tensor],
                running_mean: Optional[torch.Tensor], running_var: Optional[torch.Tensor], training: bool,
                eps: float) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """y (N, C, H, W) -> (out, mean, var): out the contiguous (N, n, H, W) fp32 ``conv2d(relu(batch_norm(y)), w1, b1)`` with w1 (n, C,
    1, 1) and b1 (n,); mean and the biased var the (C,) fp32 statistics used (the batch's when ``training``, else copies of
    ``running_mean`` / ``running_var``).  relu(batch_norm(y)) is never stored.  Bit-reproducible."""
    from .decoder import forward
    return forward(y, w1, b1, bn_weight, bn_bias, running_mean, running_var, training, eps)


@output_head.register_fake
def _(y, w1, b1, bn_weight, bn_bias, running_mean, running_var, training, eps):
    n, c, h, w = y.shape
    return (y.new_empty((n, w1.shape[0], h, w), dtype=torch.float32), y.new_empty((c,), dtype=torch.float32),
            y.new_empty((c,), dtype=torch.float32))


@torch.library.custom_op("fiery_b200::output_head_backward", mutates_args=(), device_types="cuda")
def output_head_backward(grad_out: torch.Tensor, y: torch.Tensor, mean: torch.Tensor, var: torch.Tensor, w1: torch.Tensor,
                         b1: torch.Tensor, bn_weight: Optional[torch.Tensor], bn_bias: Optional[torch.Tensor], training: bool, eps: float,
                         need: List[bool]) -> List[torch.Tensor]:
    """[grad_y, grad_bn_weight, grad_bn_bias, grad_w1, grad_b1] of ``output_head``, each in its input's shape and dtype; ``need`` (5
    flags in that order) says which are computed, the others come back empty.  Needs only y and the forward's (mean, var)."""
    from .decoder import backward
    g = backward(grad_out, y, mean, var, w1, b1, bn_weight, bn_bias, training, eps, need)
    likes = [y, bn_weight, bn_bias, w1, b1]
    return [_cast_back(gi, like if like is not None else y) for gi, like in zip(g, likes)]


@output_head_backward.register_fake
def _(grad_out, y, mean, var, w1, b1, bn_weight, bn_bias, training, eps, need):
    likes = [y, bn_weight, bn_bias, w1, b1]
    return [like.new_empty(like.shape) if nd and like is not None else y.new_empty((0,)) for like, nd in zip(likes, need)]


def _output_head_setup_context(ctx, inputs, output):
    y, w1, b1, bn_w, bn_b, _rm, _rv, training, eps = inputs
    _out, mean, var = output
    ctx.mark_non_differentiable(mean, var)
    ctx.args = (training, eps)
    ctx.save_for_backward(y, mean, var, w1, b1, bn_w, bn_b)


_OUTPUT_HEAD_GRAD_SLOTS = (0, 3, 4, 1, 2)          # the inputs output_head_backward's gradients belong to


def _output_head_backward(ctx, grad_out, _gm, _gv):
    y, mean, var, w1, b1, bn_w, bn_b = ctx.saved_tensors
    need = [bool(ctx.needs_input_grad[i]) for i in _OUTPUT_HEAD_GRAD_SLOTS]
    grads = [None] * 9
    if not any(need) or grad_out is None:
        return tuple(grads)
    g = torch.ops.fiery_b200.output_head_backward(grad_out, y, mean, var, w1, b1, bn_w, bn_b, *ctx.args, need)
    for slot, gi, nd in zip(_OUTPUT_HEAD_GRAD_SLOTS, g, need):
        grads[slot] = gi if nd else None
    return tuple(grads)


output_head.register_autograd(_output_head_backward, setup_context=_output_head_setup_context)
torch.library.register_autocast("fiery_b200::output_head", "cuda", torch.float32)


from . import bev_conv, causal_conv  # noqa: E402,F401  (they register first_conv and causal_conv3d through _register_conv)
