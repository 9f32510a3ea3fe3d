"""The future prediction's SpatialGRU on the project's kernels (fiery/layers/temporal.py:10-62, fiery/models/future_prediction.py).

A reference ``SpatialGRU`` runs its cell once per future frame: two ``torch.cat``s, ``conv_update`` and ``conv_reset`` over the same
concatenation, the sigmoids, ``(1 - r) * state``, ``conv_state_tilde`` (a bias-free 3x3 conv, BatchNorm2d and ReLU) and the blend, then
a ``torch.stack``.  ``torch.ops.fiery_b200.spatial_gru`` (registered in fiery_b200/ops.py; kernels in csrc/spatial_gru.cu on
csrc/causal_conv.cu's 3x3 kernels and csrc/batch_norm.cu's statistics) runs all T steps: the two gate convolutions as one
convolution with two output segments whose epilogue applies the sigmoids and writes q = (1 - r) h, the state convolution, and the
norm's apply pass computing the blend into the output frame.  Neither concatenation is built.  Its backward runs the recurrence in
reverse and the weight gradients once over all steps; everything is bit-reproducible.

``TensorCoreSpatialGRU.from_module(gru)`` adopts ``conv_update``, ``conv_reset`` and ``conv_state_tilde`` (``state_dict`` keys
unchanged) and looks them up at call time; ``install.use_tensor_core_future_prediction`` swaps it into a model.  No CPU path.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn as nn

from . import _lib
from ._lib import _require_cuda, f32
from .batch_norm import FusedSyncBatchNorm, gather, sync_group, update_running_stats

MAX_CHANNELS = 64


def unsupported_reason(x_channels: int, h_channels: int, grid_y: Optional[int] = None) -> Optional[str]:
    """None if the kernels take these shapes, else the reason (the limits of include/fiery_b200.h)."""
    if not 1 <= x_channels <= MAX_CHANNELS:
        return f"input_size = {x_channels} (the kernels take 1..{MAX_CHANNELS})"
    if not 1 <= h_channels <= MAX_CHANNELS:
        return f"hidden_size = {h_channels} (the kernels take 1..{MAX_CHANNELS})"
    if grid_y is not None and grid_y % 4:
        return f"W = {grid_y} map columns (the kernels need a multiple of 4: 16-byte TMA row pitch)"
    return None


def _desc(b: int, frames: int, x_frames: int, h: int, w: int, cx: int, ch: int, x_strides=None, training: bool = True,
          eps: float = 1e-5, bias_init: float = 0.0) -> _lib.SpatialGruDesc:
    d = _lib.SpatialGruDesc()
    d.batch, d.frames, d.x_frames, d.grid_x, d.grid_y, d.x_channels, d.h_channels = b, frames, x_frames, h, w, cx, ch
    sb, st, sc = x_strides if x_strides is not None else (x_frames * cx * h * w, cx * h * w, h * w)
    d.x_stride_b, d.x_stride_t, d.x_stride_c = sb, st, sc
    d.training, d.eps, d.bias_init = int(training), float(eps), float(bias_init)
    return d


def workspace_bytes(b: int, frames: int, x_frames: int, h: int, w: int, cx: int, ch: int) -> Tuple[int, int, int, int]:
    """(pack, saved, forward workspace, backward workspace) bytes from the C ABI (host-only; 0s for shapes outside the limits)."""
    lib = _lib.load()
    d = _desc(b, frames, x_frames, h, w, cx, ch)
    return (int(lib.fiery_spatial_gru_packed_bytes(d)), int(lib.fiery_spatial_gru_saved_bytes(d)),
            int(lib.fiery_spatial_gru_forward_workspace_bytes(d)), int(lib.fiery_spatial_gru_backward_workspace_bytes(d)))


def pack_weights(weights, x_channels: int) -> torch.Tensor:
    """[W_update, W_reset, W_state] -> the uint8 device pack of the four convolutions (both directions of the gates' and the state's)."""
    w_u, w_r, w_s = weights
    _require_cuda(w_u, "weight")
    ch = int(w_u.shape[0])
    if tuple(w_u.shape) != (ch, x_channels + ch, 3, 3) or w_r.shape != w_u.shape or w_s.shape != w_u.shape:
        raise ValueError(f"spatial GRU: weights {tuple(w_u.shape)}, {tuple(w_r.shape)}, {tuple(w_s.shape)} are not "
                         f"({ch}, {x_channels + ch}, 3, 3)")
    reason = unsupported_reason(x_channels, ch)
    if reason is not None:
        raise _lib.FieryError(f"spatial GRU: {reason}")
    gates = f32(torch.cat([w_u.detach(), w_r.detach()], 0))
    state = f32(w_s.detach())
    d = _desc(1, 1, 1, 1, 4, x_channels, ch)
    out = torch.empty(int(_lib.load().fiery_spatial_gru_packed_bytes(d)), dtype=torch.uint8, device=w_u.device)
    _lib.call("fiery_spatial_gru_pack_weights", w_u.device, d, gates.data_ptr(), state.data_ptr(), out.data_ptr())
    return out


def _packed(w_u: torch.Tensor, w_r: torch.Tensor, w_s: torch.Tensor) -> torch.Tensor:
    return _lib.packed(pack_weights, [w_u, w_r, w_s], int(w_u.shape[1] - w_u.shape[0]))


def gru_input(x: torch.Tensor) -> torch.Tensor:
    """x (b, Tx, C, H, W) as the kernels read it: fp32, 16-byte aligned, contiguous pixel planes and strides that are multiples of 4
    elements; x itself when it already is, else a contiguous fp32 copy (a map broadcast over the pixels is materialized here once)."""
    _, tx, _, h, w = x.shape
    ok = (x.dtype == torch.float32 and x.data_ptr() % 16 == 0 and (x.stride(4) == 1 or w == 1) and (x.stride(3) == w or h == 1)
          and x.stride(0) % 4 == 0 and x.stride(2) % 4 == 0 and (tx == 1 or x.stride(1) % 4 == 0))
    return x if ok else _aligned_f32(x)


def _aligned_f32(t: torch.Tensor) -> torch.Tensor:
    """t as a contiguous, 16-byte aligned fp32 tensor: t itself when it is one, else a copy (a contiguous fp32 view at an odd offset,
    e.g. a slice of a flat buffer, is copied too)"""
    if t.dtype == torch.float32 and t.is_contiguous() and t.data_ptr() % 16 == 0:
        return t
    return t.to(torch.float32, memory_format=torch.contiguous_format, copy=True)


def _per_channel(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    return f32(t.detach()) if t is not None else None


def _check(x: torch.Tensor, h0: torch.Tensor, w_u: torch.Tensor, frames: int) -> Tuple[int, ...]:
    b, tx, cx, h, w = x.shape
    ch = int(w_u.shape[0])
    if tx not in (1, frames) or tuple(h0.shape) != (b, ch, h, w):
        raise ValueError(f"spatial GRU: x {tuple(x.shape)}, h0 {tuple(h0.shape)} and {frames} steps do not match")
    reason = unsupported_reason(cx, ch, w)
    if reason is not None:
        raise _lib.FieryError(f"spatial GRU: {reason}")
    return b, tx, cx, h, w, ch


def _forward_operands(dims, x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b, frames: int, training: bool, eps: float, bias_init: float):
    """(d, x, h0, weight pack, gate biases, norm weight, norm bias, saved, workspace) as the kernels take them; hold them until the end."""
    b, tx, cx, h, w, ch = dims
    xs, hs = gru_input(x), _aligned_f32(h0)
    d = _desc(b, frames, tx, h, w, cx, ch, (xs.stride(0), xs.stride(1), xs.stride(2)), training, eps, bias_init)
    lib = _lib.load()
    saved = torch.empty(int(lib.fiery_spatial_gru_saved_bytes(d)), dtype=torch.uint8, device=x.device)
    bias = torch.empty(2 * ch, dtype=torch.float32, device=x.device)            # the two gate biases, without a map op (cat)
    bias[:ch], bias[ch:] = b_u.detach(), b_r.detach()
    ws = _lib.workspace(lib.fiery_spatial_gru_forward_workspace_bytes(d), x.device)
    return d, xs, hs, _packed(w_u, w_r, w_s), bias, _per_channel(bn_w), _per_channel(bn_b), saved, ws


def _grads(dims, device, need, bn_w, bn_b):
    """(grad_x, grad_h0, the gates' weight and bias (the update's C_h rows, then the reset's), grad_w_s, grad_bn_w, grad_bn_b) fp32, None
    where ``need`` (9 flags: x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b) does not ask or the norm has no such parameter."""
    b, tx, cx, h, w, ch = dims
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=device)  # noqa: E731
    gwg, gbg = (new(2 * ch, cx + ch, 3, 3), new(2 * ch)) if any(need[2:6]) else (None, None)
    return (new(b, tx, cx, h, w) if need[0] else None, new(b, ch, h, w) if need[1] else None, gwg, gbg,
            new(ch, cx + ch, 3, 3) if need[6] else None, new(ch) if need[7] and bn_w is not None else None,
            new(ch) if need[8] and bn_b is not None else None)


def _split_gates(g: Optional[torch.Tensor], ch: int, take):
    """The gates' (2 C_h, ...) gradient as (take(the update's rows), take(the reset's rows)); (None, None) for None."""
    return (take(g[:ch]), take(g[ch:])) if g is not None else (None, None)


def forward(x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b, running_mean, running_var, frames: int, training: bool, eps: float,
            bias_init: float):
    """(out (b, T, C_h, H, W), means (T, C_h), vars (T, C_h), saved): the SpatialGRU over ``frames`` steps; x (b, Tx, C_x, H, W) with
    Tx 1 (one frame read at every step) or T.  ``saved`` holds u, r, q and s of every step for the backward."""
    _require_cuda(x, "x")
    dims = b, _, _, h, w, ch = _check(x, h0, w_u, frames)
    if not training and (running_mean is None or running_var is None):
        raise ValueError("spatial GRU: eval mode needs running_mean and running_var")
    d, xs, hs, packed, bias, bw, bb, saved, ws = _forward_operands(dims, x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b, frames, training,
                                                                    eps, bias_init)
    rm, rv = _per_channel(running_mean), _per_channel(running_var)
    out = torch.empty((b, frames, ch, h, w), dtype=torch.float32, device=x.device)
    means = torch.empty((frames, ch), dtype=torch.float32, device=x.device)
    var = torch.empty((frames, ch), dtype=torch.float32, device=x.device)
    _lib.call("fiery_spatial_gru_forward", x.device, d, xs.data_ptr(), hs.data_ptr(), packed.data_ptr(), bias.data_ptr(), _ptr(bw),
              _ptr(bb), _ptr(rm), _ptr(rv), out.data_ptr(), saved.data_ptr(), means.data_ptr(), var.data_ptr(), ws.data_ptr())
    return out, means, var, saved


def backward(grad_out, x, h0, out, saved, means, var, w_u, w_r, w_s, bn_w, bn_b, frames: int, training: bool, eps: float,
             bias_init: float, need_x: bool, need_h0: bool, need_gates: bool, need_state: bool, need_bn: bool):
    """The gradients of ``forward`` in fp32: (grad_x (x's shape, contiguous), grad_h0, grad_w_u, grad_b_u, grad_w_r, grad_b_r,
    grad_w_s, grad_bn_w, grad_bn_b), None where not asked for."""
    dims = b, tx, cx, h, w, ch = _check(x, h0, w_u, frames)
    xs, hs = gru_input(x), _aligned_f32(h0)
    d = _desc(b, frames, tx, h, w, cx, ch, (xs.stride(0), xs.stride(1), xs.stride(2)), training, eps, bias_init)
    lib = _lib.load()
    dev = x.device
    bn_w, bn_b = _per_channel(bn_w), _per_channel(bn_b)
    gx, gh, gwg, gbg, gws, gbw, gbb = _grads(dims, dev, (need_x, need_h0) + (need_gates,) * 4 + (need_state, need_bn, need_bn), bn_w, bn_b)
    go, packed = _aligned_f32(grad_out), _packed(w_u, w_r, w_s)
    ws = _lib.workspace(lib.fiery_spatial_gru_backward_workspace_bytes(d), dev)
    _lib.call("fiery_spatial_gru_backward", dev, d, go.data_ptr(), xs.data_ptr(), hs.data_ptr(), out.data_ptr(),
              saved.data_ptr(), means.data_ptr(), var.data_ptr(), packed.data_ptr(), _ptr(bn_w), _ptr(bn_b), _ptr(gx),
              _ptr(gh), _ptr(gwg), _ptr(gbg), _ptr(gws), _ptr(gbw), _ptr(gbb), ws.data_ptr())
    (gwu, gwr), (gbu, gbr) = _split_gates(gwg, ch, torch.Tensor.clone), _split_gates(gbg, ch, torch.Tensor.clone)
    return gx, gh, gwu, gbu, gwr, gbr, gws, gbw, gbb


# ------------------------------------------------------------------------------------------------------------------------------
# the GRU with each step's statistics over a process group (its norm a FusedSyncBatchNorm): one gather per step each way.  One rank's
# passes are generators: each yields the step's (C, 3) fp64 triplet and is sent back the group's (world, C, 3), so autograd drives
# one of them with a collective (``run_steps``) and a test can drive several in lockstep.
# ------------------------------------------------------------------------------------------------------------------------------
def run_steps(steps, gather):
    """Run the generator ``steps`` to its end, answering each triplet it yields with ``gather(triplet)``; returns its result."""
    try:
        triplet = next(steps)
        while True:
            triplet = steps.send(gather(triplet))
    except StopIteration as done:
        return done.value


def sync_forward_steps(x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b, frames: int, eps: float, bias_init: float):
    """One rank's training forward over ``frames`` steps through the per-step entries (fiery_spatial_gru_forward_step_*): per step it
    yields this rank's (n, mean, M2) of s and takes the group's gathered triplets.  Returns (out, means, vars, counts, saved), counts
    (frames,) fp64 on the device, each step's group count.  A rank with batch 0 yields n = 0 and takes the group's statistics."""
    _require_cuda(x, "x")
    dims = b, _, _, h, w, ch = _check(x, h0, w_u, frames)
    dev = x.device
    means = torch.empty((frames, ch), dtype=torch.float32, device=dev)
    var = torch.empty((frames, ch), dtype=torch.float32, device=dev)
    counts = torch.empty(frames, dtype=torch.float64, device=dev)
    out = torch.empty((b, frames, ch, h, w), dtype=torch.float32, device=dev)
    if b == 0:
        from .batch_norm import forward_gathered
        empty = torch.empty((0, ch, 1, h, w), dtype=torch.float32, device=dev)
        for t in range(frames):
            gathered = yield torch.zeros((ch, 3), dtype=torch.float64, device=dev)
            _, means[t], var[t], counts[t:t + 1] = forward_gathered(gathered, empty, bn_w, bn_b, None, eps, True)
        return out, means, var, counts, torch.empty(0, dtype=torch.uint8, device=dev)
    d, xs, hs, packed, bias, bw, bb, saved, ws = _forward_operands(dims, x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b, frames, True, eps,
                                                                    bias_init)    # ws is kept across the steps
    for t in range(frames):
        stats = torch.empty((ch, 3), dtype=torch.float64, device=dev)
        _lib.call("fiery_spatial_gru_forward_step_begin", dev, d, t, xs.data_ptr(), hs.data_ptr(), packed.data_ptr(), bias.data_ptr(),
                  out.data_ptr(), saved.data_ptr(), stats.data_ptr(), ws.data_ptr())
        gathered = yield stats
        _lib.call("fiery_spatial_gru_forward_step_end", dev, d, t, int(gathered.shape[0]), gathered.data_ptr(), hs.data_ptr(), _ptr(bw),
                  _ptr(bb), out.data_ptr(), saved.data_ptr(), means.data_ptr(), var.data_ptr(), counts[t:].data_ptr(), ws.data_ptr())
    return out, means, var, counts, saved


def sync_backward_steps(grad_out, x, h0, out, saved, means, var, w_u, w_r, w_s, bn_w, bn_b, frames: int, eps: float, bias_init: float,
                        need):
    """The gradients of ``sync_forward_steps`` (``need``: 9 flags for x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b): per step, t = T-1 ..
    0, it yields this rank's (n, S1, S2) and takes the group's gathered triplets, then runs the weight gradients.  Returns (grad_x,
    grad_h0, grad_w_u, grad_b_u, grad_w_r, grad_b_r, grad_w_s, grad_bn_w, grad_bn_b), None where not asked for; the parameter
    gradients are this rank's own (the local sums, as torch's).  With grad_h0 not asked for, the carried gradient lives in the
    workspace."""
    dims = b, tx, cx, h, w, ch = _check(x, h0, w_u, frames)
    dev = x.device
    bw, bb = _per_channel(bn_w), _per_channel(bn_b)
    gx, gh, gwg, gbg, gws, gbw, gbb = _grads(dims, dev, need, bw, bb)
    if b == 0:
        for _ in range(frames):
            yield torch.zeros((ch, 3), dtype=torch.float64, device=dev)
        for g in (gx, gh, gwg, gbg, gws, gbw, gbb):
            if g is not None:
                g.zero_()
    else:
        xs, hs = gru_input(x), _aligned_f32(h0)
        d = _desc(b, frames, tx, h, w, cx, ch, (xs.stride(0), xs.stride(1), xs.stride(2)), True, eps, bias_init)
        lib = _lib.load()
        go = _aligned_f32(grad_out) if grad_out is not None else torch.zeros_like(out)
        packed = _packed(w_u, w_r, w_s)
        ws = _lib.workspace(lib.fiery_spatial_gru_backward_workspace_bytes(d), dev)      # kept across the steps and the weights call
        for t in reversed(range(frames)):
            sums = torch.empty((ch, 3), dtype=torch.float64, device=dev)
            _lib.call("fiery_spatial_gru_backward_step_begin", dev, d, t, go.data_ptr(), hs.data_ptr(), out.data_ptr(), saved.data_ptr(),
                      means.data_ptr(), var.data_ptr(), packed.data_ptr(), _ptr(bw), _ptr(bb), _ptr(gh), sums.data_ptr(), ws.data_ptr())
            gathered = yield sums
            _lib.call("fiery_spatial_gru_backward_step_end", dev, d, t, int(gathered.shape[0]), gathered.data_ptr(), hs.data_ptr(),
                      out.data_ptr(), saved.data_ptr(), means.data_ptr(), var.data_ptr(), packed.data_ptr(), _ptr(bw), _ptr(bb), _ptr(gx),
                      _ptr(gh), ws.data_ptr())
        _lib.call("fiery_spatial_gru_backward_weights", dev, d, xs.data_ptr(), hs.data_ptr(), out.data_ptr(), saved.data_ptr(),
                  packed.data_ptr(), _ptr(gwg), _ptr(gbg), _ptr(gws), _ptr(gbw), _ptr(gbb), ws.data_ptr())
    cast = lambda g, like: g.to(like.dtype) if g is not None else None           # noqa: E731
    (gwu, gwr), (gbu, gbr) = (_split_gates(g, ch, lambda t: t.to(w_u.dtype)) for g in (gwg, gbg))
    return cast(gx, x), cast(gh, h0), gwu, gbu, gwr, gbr, cast(gws, w_s), cast(gbw, bn_w), cast(gbb, bn_b)


class SyncSpatialGRU(torch.autograd.Function):
    """The SpatialGRU in training over ``frames`` steps with each step's batch statistics over a group: ``sync_forward_steps`` and
    ``sync_backward_steps`` run with ``gather``, which maps a (C, 3) fp64 tensor to the (world, C, 3) of every rank's, in rank order.
    Returns (out, means, vars, counts): counts (frames,) fp64, each step's group count, on the device."""

    @staticmethod
    def forward(ctx, x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b, frames: int, eps: float, bias_init: float, gather):
        out, means, var, counts, saved = run_steps(
            sync_forward_steps(x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b, frames, eps, bias_init), gather)
        ctx.mark_non_differentiable(means, var, counts)
        ctx.args = (frames, eps, bias_init, gather)
        ctx.save_for_backward(x, h0, out, saved, means, var, w_u, w_r, w_s, bn_w, bn_b)
        return out, means, var, counts

    @staticmethod
    def backward(ctx, grad_out, _gm, _gv, _gc):
        x, h0, out, saved, means, var, w_u, w_r, w_s, bn_w, bn_b = ctx.saved_tensors
        frames, eps, bias_init, gather = ctx.args
        need = tuple(bool(n) for n in ctx.needs_input_grad[:9])
        if not any(need):
            return (None,) * 13
        grads = run_steps(sync_backward_steps(grad_out, x, h0, out, saved, means, var, w_u, w_r, w_s, bn_w, bn_b, frames, eps, bias_init,
                                              need), gather)
        return grads + (None,) * 4


# ------------------------------------------------------------------------------------------------------------------------------
# the 3x3 convolution on its own (fiery_conv3x3_*): the GRU's kernels with plain stores, for tests and benchmarks
# ------------------------------------------------------------------------------------------------------------------------------
def conv3x3_desc(maps: int, h: int, w: int, in_channels, out_channels) -> _lib.Conv3x3Desc:
    d = _lib.Conv3x3Desc()
    d.maps, d.grid_x, d.grid_y = maps, h, w
    d.in_channels[0], d.in_channels[1] = in_channels
    d.out_channels[0], d.out_channels[1] = out_channels
    return d


def conv3x3_pack(weight: torch.Tensor, d: _lib.Conv3x3Desc) -> torch.Tensor:
    """weight (out0 + out1, in0 + in1, 3, 3) -> the uint8 pack of both directions."""
    w = f32(weight.detach())
    out = torch.empty(int(_lib.load().fiery_conv3x3_packed_bytes(d)), dtype=torch.uint8, device=w.device)
    _lib.call("fiery_conv3x3_pack_weights", w.device, d, w.data_ptr(), out.data_ptr())
    return out


def _ptr(t: Optional[torch.Tensor]) -> int:
    return t.data_ptr() if t is not None else 0


def conv3x3_forward(d, x0, x1, packed, y0, y1) -> None:
    """[y0, y1] = conv3x3([x0, x1]): contiguous fp32 (maps, C, X, Y) tensors, the outputs overwritten; x1 / y1 None for no segment."""
    _lib.call("fiery_conv3x3_forward", x0.device, d, x0.data_ptr(), _ptr(x1), packed.data_ptr(), y0.data_ptr(), _ptr(y1))


def conv3x3_backward_data(d, gy0, gy1, packed, gx0, gx1) -> None:
    _lib.call("fiery_conv3x3_backward_data", gy0.device, d, gy0.data_ptr(), _ptr(gy1), packed.data_ptr(), gx0.data_ptr(), _ptr(gx1))


def conv3x3_backward_weight(d, x0, x1, gy, gw, workspace) -> None:
    """gw (out0 + out1, in0 + in1, 3, 3) overwritten from x0, x1 and gy, one (maps, out0 + out1, X, Y) tensor."""
    _lib.call("fiery_conv3x3_backward_weight", x0.device, d, x0.data_ptr(), _ptr(x1), gy.data_ptr(), gw.data_ptr(), workspace.data_ptr())


# ------------------------------------------------------------------------------------------------------------------------------
# module
# ------------------------------------------------------------------------------------------------------------------------------
def _is_conv3x3(conv, bias: bool) -> bool:
    return (type(conv) is nn.Conv2d and conv.kernel_size == (3, 3) and conv.stride == (1, 1) and conv.padding == (1, 1)
            and conv.dilation == (1, 1) and conv.groups == 1 and conv.padding_mode == "zeros" and (conv.bias is not None) == bias)


def module_reason(gru) -> Optional[str]:
    """None if ``gru`` (a reference SpatialGRU) is covered by the kernels, else the reason.  The map width is checked at call time."""
    cu, cr, st = getattr(gru, "conv_update", None), getattr(gru, "conv_reset", None), getattr(gru, "conv_state_tilde", None)
    if cu is None or cr is None or st is None or not hasattr(st, "conv"):
        return f"{type(gru).__name__} does not have the SpatialGRU structure"
    if not (_is_conv3x3(cu, True) and _is_conv3x3(cr, True) and _is_conv3x3(st.conv, False)):
        return "the convolutions are not 3x3 with padding 1 and stride 1 (gates with a bias, the state without)"
    norm = getattr(st, "norm", None)
    if not (type(norm) is nn.BatchNorm2d or isinstance(norm, FusedSyncBatchNorm)):
        return f"norm {type(norm).__name__} (the kernels take BatchNorm2d, or a SyncBatchNorm swapped by use_fused_sync_batch_norm)"
    if type(getattr(st, "activation", None)) is not nn.ReLU:
        return f"activation {type(getattr(st, 'activation', None)).__name__} (the kernels take ReLU)"
    cx, ch = int(gru.input_size), int(gru.hidden_size)
    if cu.in_channels != cx + ch or cu.out_channels != ch or cr.out_channels != ch or st.conv.out_channels != ch:
        return "channel counts do not match input_size and hidden_size"
    return unsupported_reason(cx, ch)


class TensorCoreSpatialGRU(nn.Module):
    """Drop-in for a reference ``SpatialGRU`` whose T steps run as ``torch.ops.fiery_b200.spatial_gru``.  It holds the reference
    module's ``conv_update``, ``conv_reset`` and ``conv_state_tilde`` under the same names (``state_dict`` keys unchanged, the
    Parameters shared) and looks them up at call time.  The norm's running statistics move once per step, in step order, as
    ``nn.BatchNorm2d`` moves them.  A norm swapped to ``FusedSyncBatchNorm`` that synchronizes in this call runs ``SyncSpatialGRU``:
    each step's statistics over its process group, one gather per step each way.  ``state=None`` starts from zeros, as the reference does.  A map whose width is not a multiple of
    4, a ``flow``, a CPU input, or a norm or activation changed after the swap (e.g. by ``SyncBatchNorm.convert_sync_batchnorm``) runs
    the reference's own forward, with one warning."""

    def __init__(self, gru):
        super().__init__()
        self.input_size, self.hidden_size, self.gru_bias_init = gru.input_size, gru.hidden_size, gru.gru_bias_init
        self.conv_update = gru.conv_update
        self.conv_reset = gru.conv_reset
        self.conv_state_tilde = gru.conv_state_tilde
        self._reference = type(gru)

    @classmethod
    def from_module(cls, gru) -> "TensorCoreSpatialGRU":
        reason = module_reason(gru)
        if reason is not None:
            raise ValueError(f"SpatialGRU not covered by the tensor-core kernels: {reason}")
        return cls(gru)

    def gru_cell(self, x, state):
        return self._reference.gru_cell(self, x, state)

    def _call_reason(self, x, flow) -> Optional[str]:
        if flow is not None:
            return "a flow (warping inside the GRU)"
        if not x.is_cuda:
            return "a CPU input"
        if x.shape[4] % 4:
            return f"W = {x.shape[4]} map columns (the kernels need a multiple of 4)"
        return module_reason(self)

    def forward(self, x, state=None, flow=None, mode="bilinear"):
        reason = self._call_reason(x, flow)
        if reason is not None:
            _lib.warn_once(("spatial_gru", reason), f"fiery_b200: SpatialGRU call not covered by the kernels ({reason}); it runs the "
                           "reference's forward")
            return self._reference.forward(self, x, state, flow, mode)
        b, frames, _, h, w = x.shape
        if state is None:
            state = torch.zeros(b, self.hidden_size, h, w, device=x.device)
        if frames > 1 and x.stride(1) == 0:
            x = x[:, :1]                              # one frame read at every step, never expanded over time
        if x.stride(4) != 1 or x.stride(3) != w:
            x = x.contiguous()                        # a map broadcast over the pixels: materialized once, read by forward and backward
        bn = self.conv_state_tilde.norm
        group = sync_group(bn) if isinstance(bn, FusedSyncBatchNorm) else None
        if group is not None:
            out, means, var, counts = SyncSpatialGRU.apply(
                x, state, self.conv_update.weight, self.conv_update.bias, self.conv_reset.weight, self.conv_reset.bias,
                self.conv_state_tilde.conv.weight, bn.weight, bn.bias, frames, bn.eps, float(self.gru_bias_init),
                lambda t: gather(t, group))
            for t in range(frames):
                update_running_stats(bn, means[t], var[t], counts[t:t + 1])
            return out
        batch_stats = bn.training or (bn.running_mean is None and bn.running_var is None)
        out, means, var, _saved = torch.ops.fiery_b200.spatial_gru(
            x, state, self.conv_update.weight, self.conv_update.bias, self.conv_reset.weight, self.conv_reset.bias,
            self.conv_state_tilde.conv.weight, bn.weight, bn.bias, None if batch_stats else bn.running_mean,
            None if batch_stats else bn.running_var, frames, batch_stats, bn.eps, float(self.gru_bias_init))
        if batch_stats:
            for t in range(frames):
                update_running_stats(bn, means[t], var[t], b * h * w)
        return out


from . import ops as _ops  # noqa: E402,F401  (registers torch.ops.fiery_b200.spatial_gru)
