"""The future prediction's Bottlenecks on the project's kernels (fiery/layers/convolutions.py:64-168, fiery/models/future_prediction.py).

A reference ``Bottleneck`` (the plain variant ``FuturePrediction`` builds) runs three cuDNN convolutions, three ``BatchNorm2d``, three
ReLUs and the skip add, and keeps every intermediate map for its backward.  ``torch.ops.fiery_b200.bottleneck`` (registered in
fiery_b200/ops.py; csrc/bottleneck.cu on the temporal entry's 1x1 GEMM, the 3x3 kernels and the batch-norm kernels) runs

    y1 = W_down x,  y2 = conv3x3(relu(bn1(y1))),  y3 = W_up relu(bn2(y2)),  out = relu(bn3(y3)) + x

where each inner norm and ReLU is applied as the next convolution reads its operand, so relu(bn1(y1)) and relu(bn2(y2)) never exist
in memory.  Its backward keeps y1, y2 and y3 only and adds the skip in the last input gradient's epilogue; everything is
bit-reproducible.

``TensorCoreBottleneck.from_module(block)`` adopts the block's ``layers`` (``state_dict`` keys unchanged) and looks them up at call
time; ``install.use_tensor_core_bottlenecks`` swaps it into a model.  No CPU path.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib
from ._lib import _require_cuda, f32
from .batch_norm import update_running_stats

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


def backward(grad_out, x, y1, y2, y3, stats, w_d, w_c, w_u, norm_params: List[Optional[torch.Tensor]], training: bool, eps: float,
             need: List[bool]):
    """The gradients of ``forward`` in fp32, None where ``need`` (10 flags: x, W_down, W_conv, W_up, then each norm's weight and
    bias) does not ask or the norm has no such parameter: [grad_x, grad_W_down, grad_W_conv, grad_W_up, gw1, gb1, gw2, gb2, gw3, gb3]."""
    n, c, h, w = _check(x, w_d)
    m = c // 2
    dev = x.device
    xs, go = _aligned_f32(x), _aligned_f32(grad_out)
    params = [f32(p.detach()) if p is not None else None for p in norm_params]
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)  # noqa: E731
    gx = new(n, c, h, w) if need[0] else None
    gwd, gwc, gwu = (new(*wt.shape) if nd else None for wt, nd in zip((w_d, w_c, w_u), need[1:4]))
    chans = (m, m, c)
    gnorm = [new(chans[i // 2]) if need[4 + i] and params[4 * (i // 2) + i % 2] is not None else None for i in range(6)]
    d = desc(n, h, w, c, training, eps)
    lib = _lib.load()
    ws = _lib.workspace(lib.fiery_bottleneck_backward_workspace_bytes(d), dev)
    _lib.call("fiery_bottleneck_backward", dev, d, go.data_ptr(), xs.data_ptr(), y1.data_ptr(), y2.data_ptr(), y3.data_ptr(),
              stats.data_ptr(), _packed(w_d, w_c, w_u).data_ptr(), _pointers(params), _ptr(gx), _ptr(gwd), _ptr(gwc), _ptr(gwu),
              _pointers(gnorm), ws.data_ptr())
    return [gx, gwd, gwc, gwu] + gnorm


# ------------------------------------------------------------------------------------------------------------------------------
# module
# ------------------------------------------------------------------------------------------------------------------------------
def _is_conv(conv, k: int, cin: int, cout: int) -> bool:
    return (type(conv) is nn.Conv2d and conv.kernel_size == (k, k) and conv.stride == (1, 1) and conv.padding == ((k - 1) // 2,) * 2
            and conv.dilation == (1, 1) and conv.groups == 1 and conv.padding_mode == "zeros" and conv.bias is None
            and conv.in_channels == cin and conv.out_channels == cout)


def _norm_act_reason(abn, where: str) -> Optional[str]:
    if not (isinstance(abn, nn.Sequential) and len(abn) == 2):
        return f"{where} is not (BatchNorm2d, ReLU)"
    if type(abn[0]) is not nn.BatchNorm2d:
        return f"{where} norm {type(abn[0]).__name__} (the kernels take BatchNorm2d)"
    if type(abn[1]) is not nn.ReLU:
        return f"{where} activation {type(abn[1]).__name__} (the kernels take ReLU)"
    return None


def module_reason(block) -> Optional[str]:
    """None if ``block`` (a reference Bottleneck) is the plain variant the kernels cover, else the reason.  The map width is checked
    at call time."""
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
        reason = _norm_act_reason(getattr(layers, name), name)
        if reason is not None:
            return reason
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
    momentum None).  A CPU input, a map width that is not a multiple of 4, norms that disagree on batch or running statistics or on
    eps, or a norm, activation or dropout changed after the swap (e.g. by ``SyncBatchNorm.convert_sync_batchnorm``) run the
    reference's own forward, with one warning."""

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
        batch_stats = _batch_stats(norms[0])
        params = []
        for bn in norms:
            params += [bn.weight, bn.bias, None if batch_stats else bn.running_mean, None if batch_stats else bn.running_var]
        out, _y1, _y2, _y3, stats = torch.ops.fiery_b200.bottleneck(
            x, layers.conv_down_project.weight, layers.conv.weight, layers.conv_up_project.weight, *params, batch_stats, float(norms[0].eps))
        if batch_stats:
            n, c, h, w = x.shape
            m = c // 2
            offs = (0, 2 * m, 4 * m)
            for bn, o, k in zip(norms, offs, (m, m, c)):
                update_running_stats(bn, stats[o:o + k], stats[o + k:o + 2 * k], n * h * w)
        return out


from . import ops as _ops  # noqa: E402,F401  (registers torch.ops.fiery_b200.bottleneck)
