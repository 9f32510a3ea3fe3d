"""The future prediction's Bottlenecks on the project's kernels (fiery/layers/convolutions.py:64-168, fiery/models/future_prediction.py).

A reference ``Bottleneck`` (the plain variant ``FuturePrediction`` builds) runs three cuDNN convolutions, three ``BatchNorm2d``, three
ReLUs and the skip add, and keeps every intermediate map for its backward.  ``torch.ops.fiery_b200.bottleneck`` (registered in
fiery_b200/ops.py; csrc/bottleneck.cu on the temporal entry's 1x1 GEMM, the 3x3 kernels and the batch-norm kernels) runs

    y1 = W_down x,  y2 = conv3x3(relu(bn1(y1))),  y3 = W_up relu(bn2(y2)),  out = relu(bn3(y3)) + x

where each inner norm and ReLU is applied as the next convolution reads its operand, so relu(bn1(y1)) and relu(bn2(y2)) never exist
in memory.  Its backward keeps y1, y2 and y3 only and adds the skip in the last input gradient's epilogue; everything is
bit-reproducible.

``TensorCoreBottleneck.from_module(block)`` adopts the block's ``layers`` (``state_dict`` keys unchanged) and looks them up at call
time; ``install.use_tensor_core_bottlenecks`` swaps it into a model.  Under ``SyncBatchNorm`` (``install.use_tensor_core_sync_bottlenecks``
swaps the three norms for ``FusedSyncBatchNorm``s) the same chain runs in four stages split at the norms, each norm's statistics
gathered over the process group between two stages (``SyncBottleneck``).  No CPU path.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib
from ._lib import _require_cuda, f32
from .batch_norm import FusedSyncBatchNorm, _check_gathered, forward_gathered, gather, sync_group, update_running_stats
from .future_prediction import run_steps

MAX_CHANNELS = 128
_LAYERS = ("conv_down_project", "abn_down_project", "conv", "abn", "conv_up_project", "abn_up_project", "dropout")


def unsupported_reason(channels: int, grid_y: Optional[int] = None) -> Optional[str]:
    """None if the kernels take these shapes, else the reason (the limits of include/fiery_b200.h)."""
    if not 2 <= channels <= MAX_CHANNELS:
        return f"in_channels = {channels} (the kernels take 2..{MAX_CHANNELS})"
    if grid_y is not None and grid_y % 4:
        return f"W = {grid_y} map columns (the kernels need a multiple of 4: 16-byte TMA row pitch)"
    return None


def desc(maps: int, h: int, w: int, channels: int, training: bool = True, eps: float = 1e-5) -> _lib.BottleneckDesc:
    d = _lib.BottleneckDesc()
    d.maps, d.grid_x, d.grid_y, d.channels, d.training, d.eps = maps, h, w, channels, int(training), float(eps)
    return d


def workspace_bytes(maps: int, h: int, w: int, channels: int) -> Tuple[int, int, int]:
    """(pack, forward workspace, backward workspace) bytes from the C ABI (host-only; 0s for shapes outside the limits)."""
    lib = _lib.load()
    d = desc(maps, h, w, channels)
    return (int(lib.fiery_bottleneck_packed_bytes(d)), int(lib.fiery_bottleneck_forward_workspace_bytes(d)),
            int(lib.fiery_bottleneck_backward_workspace_bytes(d)))


def pack_weights(weights) -> torch.Tensor:
    """[W_down (M, C, 1, 1), W_conv (M, M, 3, 3), W_up (C, M, 1, 1)] -> the uint8 device pack of the three convolutions."""
    w_d, w_c, w_u = weights
    _require_cuda(w_d, "weight")
    c = int(w_d.shape[1])
    m = c // 2
    if tuple(w_d.shape) != (m, c, 1, 1) or tuple(w_c.shape) != (m, m, 3, 3) or tuple(w_u.shape) != (c, m, 1, 1):
        raise ValueError(f"bottleneck: weights {tuple(w_d.shape)}, {tuple(w_c.shape)}, {tuple(w_u.shape)} are not "
                         f"({m}, {c}, 1, 1), ({m}, {m}, 3, 3), ({c}, {m}, 1, 1)")
    reason = unsupported_reason(c)
    if reason is not None:
        raise _lib.FieryError(f"bottleneck: {reason}")
    ws = [f32(w.detach()) for w in weights]
    d = desc(1, 1, 4, c)
    out = torch.empty(int(_lib.load().fiery_bottleneck_packed_bytes(d)), dtype=torch.uint8, device=w_d.device)
    _lib.call("fiery_bottleneck_pack_weights", w_d.device, d, *(w.data_ptr() for w in ws), out.data_ptr())
    return out


def _packed(w_d: torch.Tensor, w_c: torch.Tensor, w_u: torch.Tensor) -> torch.Tensor:
    return _lib.packed(pack_weights, [w_d, w_c, w_u])


def _ptr(t: Optional[torch.Tensor]) -> int:
    return t.data_ptr() if t is not None else 0


def _aligned_f32(t: torch.Tensor) -> torch.Tensor:
    """t as a contiguous, 16-byte aligned fp32 tensor: t itself when it is one, else a copy."""
    if t.dtype == torch.float32 and t.is_contiguous() and t.data_ptr() % 16 == 0:
        return t
    return t.to(torch.float32, memory_format=torch.contiguous_format, copy=True)


def _pointers(ts) -> ctypes.Array:
    return (ctypes.c_void_p * len(ts))(*[_ptr(t) for t in ts])


def _check(x: torch.Tensor, w_d: torch.Tensor) -> Tuple[int, int, int, int]:
    if x.dim() != 4 or x.shape[1] != w_d.shape[1]:
        raise ValueError(f"bottleneck: x {tuple(x.shape)} is not (N, {int(w_d.shape[1])}, H, W)")
    n, c, h, w = (int(v) for v in x.shape)
    reason = unsupported_reason(c, w)
    if reason is not None:
        raise _lib.FieryError(f"bottleneck: {reason}")
    return n, c, h, w


def forward(x, w_d, w_c, w_u, norm_params: List[Optional[torch.Tensor]], training: bool, eps: float):
    """(out, y1, y2, y3, stats): the Bottleneck on x (N, C, H, W) -- out (N, C, H, W), the pre-norm maps y1, y2 (N, M, H, W) and
    y3 (N, C, H, W), and stats (2 (2M + C),) fp32, each norm's mean and biased var (copies of the running ones in eval), all fp32.
    norm_params: 12 tensors or None, norm i's weight, bias, running_mean, running_var at [4i .. 4i + 3]."""
    _require_cuda(x, "x")
    n, c, h, w = _check(x, w_d)
    m = c // 2
    if not training and any(norm_params[4 * i + j] is None for i in range(3) for j in (2, 3)):
        raise ValueError("bottleneck: eval mode needs every norm's running_mean and running_var")
    xs = _aligned_f32(x)
    params = [f32(p.detach()) if p is not None else None for p in norm_params]
    d = desc(n, h, w, c, training, eps)
    lib = _lib.load()
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=x.device)  # noqa: E731
    out, y1, y2, y3, stats = new(n, c, h, w), new(n, m, h, w), new(n, m, h, w), new(n, c, h, w), new(4 * m + 2 * c)
    ws = _lib.workspace(lib.fiery_bottleneck_forward_workspace_bytes(d), x.device)
    _lib.call("fiery_bottleneck_forward", x.device, d, xs.data_ptr(), _packed(w_d, w_c, w_u).data_ptr(), _pointers(params),
              y1.data_ptr(), y2.data_ptr(), y3.data_ptr(), out.data_ptr(), stats.data_ptr(), ws.data_ptr())
    return out, y1, y2, y3, stats


def _grad_outputs(x, weights, params, need):
    """(grad_x, grad_W_down, grad_W_conv, grad_W_up, [the norms' 6 gradients]) fp32 outputs, None where ``need`` does not ask or the
    norm has no such parameter (``params``: the norms' 12)."""
    n, c, h, w = x.shape
    m = c // 2
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=x.device)  # noqa: E731
    gx = new(n, c, h, w) if need[0] else None
    gwd, gwc, gwu = (new(*wt.shape) if nd else None for wt, nd in zip(weights, need[1:4]))
    chans = (m, m, c)
    gnorm = [new(chans[i // 2]) if need[4 + i] and params[4 * (i // 2) + i % 2] is not None else None for i in range(6)]
    return gx, gwd, gwc, gwu, gnorm


def backward(grad_out, x, y1, y2, y3, stats, w_d, w_c, w_u, norm_params: List[Optional[torch.Tensor]], training: bool, eps: float,
             need: List[bool]):
    """The gradients of ``forward`` in fp32, None where ``need`` (10 flags: x, W_down, W_conv, W_up, then each norm's weight and
    bias) does not ask or the norm has no such parameter: [grad_x, grad_W_down, grad_W_conv, grad_W_up, gw1, gb1, gw2, gb2, gw3, gb3]."""
    n, c, h, w = _check(x, w_d)
    dev = x.device
    xs, go = _aligned_f32(x), _aligned_f32(grad_out)
    params = [f32(p.detach()) if p is not None else None for p in norm_params]
    gx, gwd, gwc, gwu, gnorm = _grad_outputs(x, (w_d, w_c, w_u), params, need)
    d = desc(n, h, w, c, training, eps)
    lib = _lib.load()
    ws = _lib.workspace(lib.fiery_bottleneck_backward_workspace_bytes(d), dev)
    _lib.call("fiery_bottleneck_backward", dev, d, go.data_ptr(), xs.data_ptr(), y1.data_ptr(), y2.data_ptr(), y3.data_ptr(),
              stats.data_ptr(), _packed(w_d, w_c, w_u).data_ptr(), _pointers(params), _ptr(gx), _ptr(gwd), _ptr(gwc), _ptr(gwu),
              _pointers(gnorm), ws.data_ptr())
    return [gx, gwd, gwc, gwu] + gnorm


# ------------------------------------------------------------------------------------------------------------------------------
# the Bottleneck with its norms' statistics over a process group (its norms FusedSyncBatchNorms): one gather per norm each way.  One
# rank's passes are generators, as future_prediction.sync_forward_steps: each yields the norm's (channels, 3) fp64 triplet and is sent
# back the group's (world, channels, 3), so autograd drives one of them with a collective (``run_steps``) and a test several in lockstep.
# ------------------------------------------------------------------------------------------------------------------------------
def _stats_slices(m: int, c: int):
    """(offset, channels) of each norm's mean in ``forward``'s stats; its var follows at offset + channels."""
    return ((0, m), (2 * m, m), (4 * m, c))


def sync_forward_stages(x, w_d, w_c, w_u, norm_params: List[Optional[torch.Tensor]], eps: float):
    """One rank's training forward through fiery_bottleneck_sync_forward_stage: after stages 0, 1 and 2 it yields this rank's (n, mean,
    M2) of y1, y2 and y3 and takes the group's gathered triplets.  norm_params: 6 tensors or None, norm i's weight and bias at [2i],
    [2i + 1].  Returns (out, y1, y2, y3, stats, counts): as ``forward``'s, and counts (3,) fp64 on the device, each norm's group count.
    A rank with no maps yields n = 0 three times and takes the group's statistics (the batch-norm group entries)."""
    _require_cuda(x, "x")
    n, c, h, w = _check(x, w_d)
    m = c // 2
    dev = x.device
    params = [f32(p.detach()) if p is not None else None for p in norm_params]
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)  # noqa: E731
    out, y1, y2, y3, stats = new(n, c, h, w), new(n, m, h, w), new(n, m, h, w), new(n, c, h, w), new(4 * m + 2 * c)
    counts = torch.empty(3, dtype=torch.float64, device=dev)
    if n == 0:
        for i, (o, k) in enumerate(_stats_slices(m, c)):
            gathered = yield torch.zeros((k, 3), dtype=torch.float64, device=dev)
            empty = torch.empty((0, k, 1, h, w), dtype=torch.float32, device=dev)
            _, stats[o:o + k], stats[o + k:o + 2 * k], counts[i:i + 1] = forward_gathered(gathered, empty, params[2 * i], params[2 * i + 1],
                                                                                           None, eps, True)
        return out, y1, y2, y3, stats, counts
    xs = _aligned_f32(x)
    d = desc(n, h, w, c, True, eps)
    ws = _lib.workspace(_lib.load().fiery_bottleneck_forward_workspace_bytes(d), dev)         # kept from stage 0 to stage 3
    packed = _packed(w_d, w_c, w_u)
    norms = _pointers([params[0], params[1], None, None, params[2], params[3], None, None, params[4], params[5], None, None])
    gathered = None
    for stage, y in enumerate((y1, y2, y3, None)):
        if gathered is not None:
            _check_gathered(gathered, (y1, y2, y3)[stage - 1])
        local = torch.empty((y.shape[1], 3), dtype=torch.float64, device=dev) if y is not None else None
        _lib.call("fiery_bottleneck_sync_forward_stage", dev, d, stage, int(gathered.shape[0]) if gathered is not None else 1,
                  _ptr(gathered), xs.data_ptr(), packed.data_ptr(), norms, y1.data_ptr(), y2.data_ptr(), y3.data_ptr(), out.data_ptr(),
                  stats.data_ptr(), counts.data_ptr(), _ptr(local), ws.data_ptr())
        if local is not None:
            gathered = yield local
    return out, y1, y2, y3, stats, counts


def sync_stages(need, norm_params) -> int:
    """The deepest backward stage the gradients ``need`` asks for take (10 flags as ``backward``'s; ``norm_params`` the 6 weights and
    biases, a flag for a missing one asks for nothing): 3 for grad_x or grad_W_down, else 2 for grad_W_conv or norm 1's, else 1 for
    grad_W_up or norm 2's, else 0.  The backward gathers that many times; it depends on the flags only, the same on every rank."""
    asked = list(need[:4]) + [nd and p is not None for nd, p in zip(need[4:], norm_params)]
    if asked[0] or asked[1]:
        return 3
    if asked[2] or asked[4] or asked[5]:
        return 2
    return 1 if asked[3] or asked[6] or asked[7] else 0


def sync_backward_stages(grad_out, x, y1, y2, y3, stats, w_d, w_c, w_u, norm_params: List[Optional[torch.Tensor]], eps: float, need):
    """The gradients of ``sync_forward_stages`` in fp32 through fiery_bottleneck_sync_backward_stage (``need``: 10 flags as
    ``backward``'s): after stages 0 .. ``sync_stages(need, norm_params)`` - 1 it yields this rank's (n, S1, S2) of norm 3, 2, 1 and
    takes the group's gathered sums.  Returns [grad_x, grad_W_down, grad_W_conv, grad_W_up, gw1, gb1, gw2, gb2, gw3, gb3], None where
    not asked for; the norms' gradients are this rank's own (the local sums, as torch's).  A rank with no maps yields n = 0 and returns
    zero gradients."""
    n, c, h, w = _check(x, w_d)
    m = c // 2
    dev = x.device
    params = [f32(p.detach()) if p is not None else None for p in norm_params]
    gx, gwd, gwc, gwu, gnorm = _grad_outputs(x, (w_d, w_c, w_u), [params[0], params[1], None, None, params[2], params[3], None, None,
                                                                  params[4], params[5], None, None], need)
    grads = [gx, gwd, gwc, gwu] + gnorm
    last = sync_stages(need, norm_params)
    chans = (c, m, m)                                             # norm 3, 2, 1: the norms of stages 0, 1, 2
    if n == 0:
        for stage in range(last):
            yield torch.zeros((chans[stage], 3), dtype=torch.float64, device=dev)
        for g in grads:
            if g is not None:
                g.zero_()
        return grads
    xs, go = _aligned_f32(x), _aligned_f32(grad_out)
    d = desc(n, h, w, c, True, eps)
    ws = _lib.workspace(_lib.load().fiery_bottleneck_backward_workspace_bytes(d), dev)        # kept from stage 0 to the last
    norms = _pointers([params[0], params[1], None, None, params[2], params[3], None, None, params[4], params[5], None, None])
    packed = _packed(w_d, w_c, w_u)
    gathered = None
    for stage in range(last + 1):
        if gathered is not None:
            _check_gathered(gathered, (y3, y2, y1)[stage - 1])
        local = torch.empty((chans[stage], 3), dtype=torch.float64, device=dev) if stage < 3 else None
        _lib.call("fiery_bottleneck_sync_backward_stage", dev, d, stage, int(gathered.shape[0]) if gathered is not None else 1,
                  _ptr(gathered), go.data_ptr(), xs.data_ptr(), y1.data_ptr(), y2.data_ptr(), y3.data_ptr(), stats.data_ptr(),
                  packed.data_ptr(), norms, _ptr(gx), _ptr(gwd), _ptr(gwc), _ptr(gwu), _pointers(gnorm), _ptr(local), ws.data_ptr())
        if stage < last:
            gathered = yield local
    return grads


class SyncBottleneck(torch.autograd.Function):
    """The Bottleneck in training with each norm's batch statistics over a group: ``sync_forward_stages`` and ``sync_backward_stages``
    run with ``gather``, which maps a (C, 3) fp64 tensor to the (world, C, 3) of every rank's, in rank order.  fp32 whatever the
    inputs' dtypes (under autocast too, as ``torch.ops.fiery_b200.bottleneck``), the gradients in the inputs' dtypes.  Returns (out,
    stats, counts): stats ``forward``'s, counts (3,) fp64 each norm's group count, on the device; neither differentiable."""

    @staticmethod
    def forward(ctx, x, w_d, w_c, w_u, n1w, n1b, n2w, n2b, n3w, n3b, eps: float, gather):
        out, y1, y2, y3, stats, counts = run_steps(sync_forward_stages(x, w_d, w_c, w_u, [n1w, n1b, n2w, n2b, n3w, n3b], eps), gather)
        ctx.mark_non_differentiable(stats, counts)
        ctx.eps, ctx.gather = eps, gather
        ctx.save_for_backward(x, y1, y2, y3, stats, w_d, w_c, w_u, n1w, n1b, n2w, n2b, n3w, n3b)
        return out, stats, counts

    @staticmethod
    def backward(ctx, grad_out, _gs, _gc):
        x, y1, y2, y3, stats, w_d, w_c, w_u, *norm_params = ctx.saved_tensors
        need = [bool(nd) for nd in ctx.needs_input_grad[:10]]
        if not any(need):
            return (None,) * 12
        grads = run_steps(sync_backward_stages(grad_out, x, y1, y2, y3, stats, w_d, w_c, w_u, norm_params, ctx.eps, need), ctx.gather)
        likes = [x, w_d, w_c, w_u] + norm_params
        return tuple(g.to(like.dtype) if g is not None else None for g, like in zip(grads, likes)) + (None, None)


# ------------------------------------------------------------------------------------------------------------------------------
# module
# ------------------------------------------------------------------------------------------------------------------------------
def _is_conv(conv, k: int, cin: int, cout: int) -> bool:
    return (type(conv) is nn.Conv2d and conv.kernel_size == (k, k) and conv.stride == (1, 1) and conv.padding == ((k - 1) // 2,) * 2
            and conv.dilation == (1, 1) and conv.groups == 1 and conv.padding_mode == "zeros" and conv.bias is None
            and conv.in_channels == cin and conv.out_channels == cout)


# the norms a block may hold, all three of one kind: BatchNorm2d, or a SyncBatchNorm swapped by use_tensor_core_sync_bottlenecks
NORM_KINDS = (nn.BatchNorm2d, FusedSyncBatchNorm)


def _norm_act_reason(abn, where: str, kinds) -> Optional[str]:
    if not (isinstance(abn, nn.Sequential) and len(abn) == 2):
        return f"{where} is not (BatchNorm2d, ReLU)"
    if type(abn[0]) not in kinds:
        return f"{where} norm {type(abn[0]).__name__} (the kernels take {' or '.join(k.__name__ for k in kinds)})"
    if type(abn[1]) is not nn.ReLU:
        return f"{where} activation {type(abn[1]).__name__} (the kernels take ReLU)"
    return None


def module_reason(block, kinds=NORM_KINDS) -> Optional[str]:
    """None if ``block`` (a reference Bottleneck) is the plain variant the kernels cover, its three norms of one of ``kinds``, else
    the reason.  The map width is checked at call time."""
    layers = getattr(block, "layers", None)
    if not isinstance(layers, nn.Sequential) or tuple(layers._modules) != _LAYERS:
        return f"{type(block).__name__} does not have the Bottleneck structure"
    if getattr(block, "projection", None) is not None:
        return "a skip projection (downsample, upsample or out_channels != in_channels)"
    c = int(getattr(layers.conv_down_project, "in_channels", 0))
    m = c // 2
    if not _is_conv(layers.conv_down_project, 1, c, m) or not _is_conv(layers.conv_up_project, 1, m, c):
        return "the projections are not bias-free 1x1 convolutions C -> C / 2 -> C"
    if not _is_conv(layers.conv, 3, m, m):
        return "the bottleneck convolution is not a bias-free 3x3 Conv2d with padding 1 and stride 1"
    for name in ("abn_down_project", "abn", "abn_up_project"):
        reason = _norm_act_reason(getattr(layers, name), name, kinds)
        if reason is not None:
            return reason
    if len({type(bn) for bn in _norms(layers)}) != 1:
        return "norms of different kinds (the kernels take three BatchNorm2d or three FusedSyncBatchNorm)"
    if not (type(layers.dropout) is nn.Dropout2d and layers.dropout.p == 0):
        return f"dropout {type(layers.dropout).__name__}(p = {getattr(layers.dropout, 'p', None)}) (the kernels take Dropout2d with p = 0)"
    return unsupported_reason(c)


def _norms(layers) -> Tuple[nn.BatchNorm2d, nn.BatchNorm2d, nn.BatchNorm2d]:
    return layers.abn_down_project[0], layers.abn[0], layers.abn_up_project[0]


def _batch_stats(bn) -> bool:
    return bn.training or (bn.running_mean is None and bn.running_var is None)


class TensorCoreBottleneck(nn.Module):
    """Drop-in for a reference ``Bottleneck`` (the plain variant) whose forward runs as ``torch.ops.fiery_b200.bottleneck``.  It holds
    the reference module's ``layers`` under the same name (``state_dict`` keys unchanged, the Parameters shared) and looks them up
    at call time.  Each norm's running statistics move as ``nn.BatchNorm2d`` moves them (momentum, or the cumulative average for
    momentum None).  Norms swapped to ``FusedSyncBatchNorm`` that synchronize in this call (one process group for all three) run
    ``SyncBottleneck``: each norm's statistics over the group, one gather per norm each way; otherwise they compute what BatchNorm2d
    norms would.  A CPU input, a map width that is not a multiple of 4, norms that disagree on batch or running statistics, on eps or
    on the process group they synchronize over, or a norm, activation or dropout changed after the swap (e.g. by
    ``SyncBatchNorm.convert_sync_batchnorm``) run the reference's own forward, with one warning."""

    def __init__(self, block):
        super().__init__()
        self.layers = block.layers
        self.projection = None
        self._downsample = getattr(block, "_downsample", False)
        self._reference = type(block)

    @classmethod
    def from_module(cls, block) -> "TensorCoreBottleneck":
        reason = module_reason(block)
        if reason is not None:
            raise ValueError(f"Bottleneck not covered by the tensor-core kernels: {reason}")
        return cls(block)

    def _call_reason(self, x) -> Optional[str]:
        if not x.is_cuda:
            return "a CPU input"
        if x.dim() != 4:
            return f"a {x.dim()}-D input (the kernels take (N, C, H, W))"
        if x.shape[3] % 4:
            return f"W = {x.shape[3]} map columns (the kernels need a multiple of 4)"
        reason = module_reason(self)
        if reason is not None:
            return reason
        norms = _norms(self.layers)
        if len({_batch_stats(bn) for bn in norms}) != 1:
            return "norms that disagree on batch or running statistics"
        if len({float(bn.eps) for bn in norms}) != 1:
            return "norms with different eps"
        if isinstance(norms[0], FusedSyncBatchNorm) and len({id(sync_group(bn)) for bn in norms}) != 1:
            return "norms that synchronize over different process groups"
        return None

    def forward(self, *args):
        (x,) = args
        reason = self._call_reason(x)
        if reason is not None:
            _lib.warn_once(("bottleneck", reason), f"fiery_b200: Bottleneck call not covered by the kernels ({reason}); it runs the "
                           "reference's forward")
            return self._reference.forward(self, x)
        layers = self.layers
        norms = _norms(layers)
        group = sync_group(norms[0]) if isinstance(norms[0], FusedSyncBatchNorm) else None
        if group is not None:
            _require_cuda(x, "x")
            out, stats, counts = SyncBottleneck.apply(x, layers.conv_down_project.weight, layers.conv.weight, layers.conv_up_project.weight,
                                                      *(p for bn in norms for p in (bn.weight, bn.bias)), float(norms[0].eps),
                                                      lambda t: gather(t, group))
            m = x.shape[1] // 2
            for i, (bn, (o, k)) in enumerate(zip(norms, _stats_slices(m, x.shape[1]))):
                update_running_stats(bn, stats[o:o + k], stats[o + k:o + 2 * k], counts[i:i + 1])
            return out
        batch_stats = _batch_stats(norms[0])
        params = []
        for bn in norms:
            params += [bn.weight, bn.bias, None if batch_stats else bn.running_mean, None if batch_stats else bn.running_var]
        out, _y1, _y2, _y3, stats = torch.ops.fiery_b200.bottleneck(
            x, layers.conv_down_project.weight, layers.conv.weight, layers.conv_up_project.weight, *params, batch_stats, float(norms[0].eps))
        if batch_stats:
            n, c, h, w = x.shape
            for bn, (o, k) in zip(norms, _stats_slices(c // 2, c)):
                update_running_stats(bn, stats[o:o + k], stats[o + k:o + 2 * k], n * h * w)
        return out


from . import ops as _ops  # noqa: E402,F401  (registers torch.ops.fiery_b200.bottleneck)
