"""The temporal block's input projections on the tensor cores (fiery/layers/temporal.py:218-281).

A reference ``TemporalBlock`` applies four 1x1x1 ``Conv3d`` to the same input -- ``convolution_paths[0][0].conv``,
``convolution_paths[1][0].conv``, ``convolution_paths[2].conv`` (each in -> in / 2) and ``projection[0]`` (in -> out, when the block
changes the channel count) -- so they are one GEMM over the input's pixel planes.  ``torch.ops.fiery_b200.temporal_entry``
(fiery_b200/ops.py; kernels in csrc/temporal_entry.cu) computes it: it reads the input as it lies (the permuted view
``TemporalModel.forward`` makes, or a contiguous NCDHW tensor) and writes each conv's output as its own contiguous
(b, C, s, X, Y) tensor, the layout ``BatchNorm3d`` and the causal convolutions take.  Both gradients run on the tensor cores too;
the weight gradient is bit-reproducible.

``TensorCoreTemporalBlock.from_block(block)`` adopts the reference block's children under the same names (``state_dict`` keys are
unchanged) and replaces only those four convolutions; ``install.use_tensor_core_temporal_model`` swaps it into a model.

``temporal_model_forward(temporal_model, bev, future_egomotion)`` is the folded form of fiery.py:148-158: the egopose channels
are constant over the map, so instead of concatenating them to the BEV (a 70-channel copy) the first block's GEMM takes the 64-channel
BEV and the egopose enters as a per-(frame, output channel) bias; its pyramid pooling is computed from the BEV's spatial means and the
egopose itself.  No CPU path.

``TensorCorePyramidPooling`` (swapped in by ``install.use_tensor_core_pyramid_pooling``) computes the block's pyramid pooling from the
input's spatial sums (``torch.ops.fiery_b200.spatial_sums``, csrc/spatial_sums.cu).  With it, a ``TensorCoreTemporalBlock`` runs its
aggregation conv as ``torch.ops.fiery_b200.temporal_aggregation``: the entry's input-gradient GEMM in swapped roles with the pooled
vector as a per-(frame, output channel) bias, so neither the concat nor the broadcast over the map is built.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from . import ops as _ops  # noqa: F401  (registers torch.ops.fiery_b200.temporal_entry)
from ._lib import _require_cuda, f32, f32_planes, warn_once
from .batch_norm import norm_act

MAX_IN_CHANNELS, MAX_OUT_CHANNELS, MAX_EXTRA_CHANNELS = 128, 256, 8


def _round8(n: int) -> int:
    return (n + 7) // 8 * 8


def unsupported_reason(in_channels: int, seg_channels: Sequence[int], extra_channels: int = 0,
                       pixels: Optional[int] = None) -> Optional[str]:
    """None if the kernels take these shapes, else the reason (the limits of include/fiery_b200.h)."""
    if not 1 <= in_channels <= MAX_IN_CHANNELS:
        return f"in_channels K = {in_channels} (the kernels take 1..{MAX_IN_CHANNELS})"
    if not 0 <= extra_channels <= MAX_EXTRA_CHANNELS:
        return f"extra_channels E = {extra_channels} (the kernels take 0..{MAX_EXTRA_CHANNELS})"
    if not 1 <= len(seg_channels) <= 4:
        return f"{len(seg_channels)} convolutions (the kernels take 1..4)"
    if sum(seg_channels) > MAX_OUT_CHANNELS or sum(_round8(c) for c in seg_channels) > MAX_OUT_CHANNELS:
        return f"N_out = {sum(seg_channels)} output channels {tuple(seg_channels)} (the kernels take <= {MAX_OUT_CHANNELS})"
    if pixels is not None and pixels % 4:
        return f"X*Y = {pixels} pixels (the kernels need a multiple of 4: 16-byte TMA pitch)"
    return None


def _desc(x: torch.Tensor, seg_channels: Sequence[int], extra_channels: int) -> _lib.TemporalEntryDesc:
    b, k, s, h, w = x.shape
    d = _lib.TemporalEntryDesc()
    d.batch, d.frames, d.pixels, d.in_channels, d.extra_channels = b, s, h * w, k, extra_channels
    d.n_segments = len(seg_channels)
    for i, c in enumerate(seg_channels):
        d.seg_channels[i] = int(c)
    d.in_stride_b, d.in_stride_c, d.in_stride_t = x.stride(0), x.stride(1), x.stride(2)
    return d


def _takes_as_is(shape, stride) -> bool:
    """The kernels read (b, K, s, X, Y) as it lies when the pixel planes are contiguous, every other stride is a multiple of 4
    elements (16-byte TMA pitch) and no two elements share an address: the input gradient is written with these strides, so an
    expanded (stride-0) or otherwise overlapping input is read from a contiguous copy instead."""
    _, _, _, h, w = shape
    if not ((stride[4] == 1 or w == 1) and (stride[3] == w or h == 1) and all(st % 4 == 0 for st in stride[:3])):
        return False
    # non-overlapping: with the dimensions of size > 1 sorted by stride, each stride covers the extent of the one before it
    dims = sorted((st, n) for st, n in zip(stride, shape) if n > 1)
    extent = 1
    for st, n in dims:
        if st < extent:
            return False
        extent = st * n
    return True


def input_strides(shape, stride) -> Tuple[int, ...]:
    """Strides of the tensor the kernels read for an input of this shape / stride: its own, or those of a contiguous copy.  The input
    gradient comes back with these strides."""
    if _takes_as_is(shape, stride):
        return tuple(stride)
    b, k, s, h, w = shape
    return (k * s * h * w, s * h * w, h * w, w, 1)


def _entry_input(x: torch.Tensor) -> torch.Tensor:
    x = x.float() if x.dtype != torch.float32 else x
    return x if _takes_as_is(x.shape, x.stride()) else x.contiguous()


def _stacked(weights: Sequence[torch.Tensor]) -> torch.Tensor:
    return torch.cat([w.detach().float().reshape(w.shape[0], -1) for w in weights], 0).contiguous()


def pack_weights(weights: Sequence[torch.Tensor], in_channels: int) -> torch.Tensor:
    """(C_q, K + E, 1, 1, 1) conv weights -> the uint8 device pack the three kernels take."""
    _require_cuda(weights[0], "weight")
    lib = _lib.load()
    w = _stacked(weights)
    seg = [int(t.shape[0]) for t in weights]
    d = _desc(torch.empty((0, in_channels, 0, 1, 4)), seg, w.shape[1] - in_channels)
    n = int(lib.fiery_temporal_entry_packed_bytes(d))
    if n == 0:
        raise _lib.FieryError(f"temporal entry: weights {[tuple(t.shape) for t in weights]} with K = {in_channels} are not supported: "
                              f"{unsupported_reason(in_channels, seg, w.shape[1] - in_channels)}")
    out = torch.empty(n, dtype=torch.uint8, device=w.device)
    _lib.call("fiery_temporal_entry_pack_weights", w.device, d, w.data_ptr(), out.data_ptr())
    return out


def _ptrs(ts: Sequence[torch.Tensor]):
    arr = (_lib.c_void_p * 4)()
    for i, t in enumerate(ts):
        arr[i] = t.data_ptr()
    return arr


def entry_forward(x: torch.Tensor, weights: Sequence[torch.Tensor], extra: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
    """x (b, K, s, X, Y) any float dtype and strides; weights: 1..4 tensors (C_q, K + E, 1, 1, 1); extra: (b, s, E) or None.  Returns
    the C_q-channel outputs, each a contiguous (b, C_q, s, X, Y) fp32 tensor."""
    _require_cuda(x, "x")
    xs = _entry_input(x)
    b, K, s, h, w = xs.shape
    seg = [int(t.shape[0]) for t in weights]
    E = int(weights[0].shape[1]) - K
    reason = unsupported_reason(K, seg, E, h * w)
    if reason is not None:
        raise _lib.FieryError(f"temporal entry: {reason}")
    outs = [torch.empty((b, c, s, h, w), dtype=torch.float32, device=x.device) for c in seg]
    e = f32(extra.detach()) if E and extra is not None else None
    if E and (e is None or tuple(e.shape) != (b, s, E)):
        raise ValueError(f"extra must be ({b}, {s}, {E}) for weights with {K + E} input channels and x with {K}")
    packed = _lib.packed(pack_weights, weights, K)
    _lib.call("fiery_temporal_entry_forward", x.device, _desc(xs, seg, E), xs.data_ptr(), e.data_ptr() if e is not None else 0,
              packed.data_ptr(), _ptrs(outs))
    return outs


def entry_backward_data(grads: Sequence[torch.Tensor], x: torch.Tensor, weights: Sequence[torch.Tensor]) -> torch.Tensor:
    """The input gradient: x's shape in fp32, with ``input_strides(x)``."""
    b, K, s, h, w = x.shape
    seg = [int(t.shape[0]) for t in weights]
    E = int(weights[0].shape[1]) - K
    gs = [f32(g) for g in grads]
    gx = torch.empty_strided(tuple(x.shape), input_strides(x.shape, x.stride()), dtype=torch.float32, device=x.device)
    packed = _lib.packed(pack_weights, weights, K)
    _lib.call("fiery_temporal_entry_backward_data", x.device, _desc(gx, seg, E), _ptrs(gs), packed.data_ptr(), gx.data_ptr())
    return gx


def backward_weight_workspace_bytes(x_shape, seg_channels: Sequence[int], extra_channels: int = 0) -> int:
    """Bytes of device workspace the weight gradient uses (host-only answer; 0 for 0 frames or unsupported shapes)."""
    b, k, s, h, w = x_shape
    return int(_lib.load().fiery_temporal_entry_backward_weight_workspace_bytes(
        _desc(torch.empty((b, k, s, h, w), device="meta"), seg_channels, extra_channels)))


def entry_backward_weight(grads: Sequence[torch.Tensor], x: torch.Tensor, weights: Sequence[torch.Tensor],
                          extra: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
    """The weight gradients, each of its weight's shape in fp32; bit-reproducible (fixed summation order, no atomics)."""
    lib = _lib.load()
    xs = _entry_input(x)
    K = xs.shape[1]
    seg = [int(t.shape[0]) for t in weights]
    E = int(weights[0].shape[1]) - K
    gs = [f32(g) for g in grads]
    e = f32(extra.detach()) if E and extra is not None else None
    d = _desc(xs, seg, E)
    ws = _lib.workspace(lib.fiery_temporal_entry_backward_weight_workspace_bytes(d), x.device)
    gw = torch.empty((sum(seg), K + E), dtype=torch.float32, device=x.device)
    _lib.call("fiery_temporal_entry_backward_weight", x.device, d, xs.data_ptr(), e.data_ptr() if e is not None else 0, _ptrs(gs),
              gw.data_ptr(), ws.data_ptr())
    return [g.reshape(t.shape).clone() for g, t in zip(gw.split(seg, 0), weights)]     # separate tensors: operator outputs may not alias


# ------------------------------------------------------------------------------------------------------------------------------
# spatial sums and the temporal aggregation (csrc/spatial_sums.cu; csrc/temporal_entry.cu in swapped roles)
# ------------------------------------------------------------------------------------------------------------------------------
def spatial_sums(x: torch.Tensor) -> torch.Tensor:
    """x (b, C, s, X, Y) any float dtype -> (b, C, s) fp32 sums over each pixel plane, in a summation order that depends on X*Y only.
    Read as it lies when x is fp32 with contiguous pixel planes (any b / C / s strides), else from a contiguous fp32 copy."""
    _require_cuda(x, "x")
    b, c, s, h, w = x.shape
    xs = f32_planes(x)
    out = torch.empty((b, c, s), dtype=torch.float32, device=x.device)
    d = _lib.SpatialSumsDesc()
    d.batch, d.channels, d.frames, d.pixels = b, c, s, h * w
    d.stride_b, d.stride_c, d.stride_t = xs.stride(0), xs.stride(1), xs.stride(2)
    _lib.call("fiery_spatial_sums", x.device, d, xs.data_ptr(), out.data_ptr())
    return out


def aggregation_reason(n_out: int, path_channels: Sequence[int], pixels: Optional[int] = None) -> Optional[str]:
    """None if the aggregation kernel takes these shapes, else the reason: the entry's input gradient in swapped roles, so N (the
    aggregation's output channels) has the entry's input limit and the paths its output limits."""
    if not 1 <= n_out <= MAX_IN_CHANNELS:
        return f"{n_out} aggregation output channels (the kernel takes 1..{MAX_IN_CHANNELS})"
    return unsupported_reason(n_out, path_channels, 0, pixels)


def _aggregation_desc(shape, path_channels: Sequence[int]) -> _lib.TemporalEntryDesc:
    """the entry descriptor in swapped roles: K = N, segments = the paths, strides of the contiguous (b, N, s, X, Y) output (or input)"""
    b, n, s, h, w = shape
    return _desc(torch.empty((b, n, s, h, w), device="meta"), path_channels, 0)


def pack_aggregation(weight: torch.Tensor, path_channels: Tuple[int, ...]) -> torch.Tensor:
    """(N, sum C_q + R, 1, 1, 1) aggregation weight -> the entry pack of its path columns, transposed: (sum C_q, N)."""
    _require_cuda(weight, "weight")
    n = int(weight.shape[0])
    wt = weight.detach().float().reshape(n, -1)[:, :sum(path_channels)].t().contiguous()
    return pack_weights([t[..., None, None, None] for t in wt.split(list(path_channels), 0)], n)


def _pooled_columns(weight: torch.Tensor, n_paths: int) -> torch.Tensor:
    n = int(weight.shape[0])
    return weight.detach().float().reshape(n, -1)[:, n_paths:]


def aggregation_forward(paths: Sequence[torch.Tensor], weight: torch.Tensor, pooled: torch.Tensor) -> torch.Tensor:
    """The aggregation conv of ``cat([*paths, pooled broadcast over the map], 1)`` without the concat: paths (b, C_q, s, X, Y), weight
    (N, sum C_q + R, 1, 1, 1), pooled (b, R, s).  Returns the contiguous (b, N, s, X, Y) fp32 output; the pooled columns enter as the
    per-(frame, output channel) bias W_P pooled, computed in fp32."""
    _require_cuda(paths[0], "paths")
    ps = [f32(p) for p in paths]
    seg = tuple(int(p.shape[1]) for p in ps)
    b, _, s, h, w = ps[0].shape
    n = int(weight.shape[0])
    if int(weight.shape[1]) != sum(seg) + pooled.shape[1] or tuple(pooled.shape) != (b, int(weight.shape[1]) - sum(seg), s):
        raise ValueError(f"temporal aggregation: paths {[tuple(p.shape) for p in ps]}, pooled {tuple(pooled.shape)} and weight "
                         f"{tuple(weight.shape)} do not match")
    reason = aggregation_reason(n, seg, h * w)
    if reason is not None:
        raise _lib.FieryError(f"temporal aggregation: {reason}")
    # bias[b, t, o] = sum_r W_P[o, r] pooled[b, r, t]: elementwise products and a sum, fp32 whatever the matmul precision setting
    wp = _pooled_columns(weight, sum(seg))
    bias = (f32(pooled).permute(0, 2, 1)[:, :, None, :] * wp).sum(-1).contiguous() if wp.shape[1] else None
    out = torch.empty((b, n, s, h, w), dtype=torch.float32, device=ps[0].device)
    packed = _lib.packed(pack_aggregation, weight, seg)
    _lib.call("fiery_temporal_aggregation_forward", out.device, _aggregation_desc(out.shape, seg), _ptrs(ps), packed.data_ptr(),
              bias.data_ptr() if bias is not None else 0, out.data_ptr())
    return out


def aggregation_backward(grad: torch.Tensor, paths: Sequence[torch.Tensor], weight: torch.Tensor, pooled: torch.Tensor,
                         need_paths: bool, need_weight: bool, need_pooled: bool):
    """(grad_paths, grad_weight, grad_pooled) of ``aggregation_forward``, fp32, None where not asked for.  grad_paths = A_q^T grad
    (the entry's forward with x = grad), the path columns of grad_weight = sum grad paths^T (the entry's weight gradient,
    bit-reproducible), and the pooled terms from G = the spatial sums of grad: grad_W_P = sum_{b,t} G pooled^T, grad_pooled = W_P^T G."""
    lib = _lib.load()
    g = f32(grad)
    seg = tuple(int(p.shape[1]) for p in paths)
    n, c = int(weight.shape[0]), sum(seg)
    d = _aggregation_desc(g.shape, seg)
    grad_paths = grad_weight = grad_pooled = None
    if need_paths:
        b, _, s, h, w = g.shape
        grad_paths = [torch.empty((b, cq, s, h, w), dtype=torch.float32, device=g.device) for cq in seg]
        packed = _lib.packed(pack_aggregation, weight, seg)
        _lib.call("fiery_temporal_entry_forward", g.device, d, g.data_ptr(), 0, packed.data_ptr(), _ptrs(grad_paths))
    if need_weight or need_pooled:
        sums = spatial_sums(g)                                      # (b, N, s)
        wp = _pooled_columns(weight, c)
        v = f32(pooled)
        if need_pooled:
            grad_pooled = (wp[None, :, :, None] * sums[:, :, None, :]).sum(1)
        if need_weight:
            ps = [f32(p) for p in paths]
            ws = _lib.workspace(lib.fiery_temporal_entry_backward_weight_workspace_bytes(d), g.device)
            gw = torch.empty((c, n), dtype=torch.float32, device=g.device)
            _lib.call("fiery_temporal_entry_backward_weight", g.device, d, g.data_ptr(), 0, _ptrs(ps), gw.data_ptr(), ws.data_ptr())
            grad_wp = (sums[:, :, None, :] * v[:, None, :, :]).sum((0, 3))
            grad_weight = torch.cat([gw.t(), grad_wp], 1).reshape(weight.shape)
    return grad_paths, grad_weight, grad_pooled


# ------------------------------------------------------------------------------------------------------------------------------
# module
# ------------------------------------------------------------------------------------------------------------------------------
def _is_1x1x1(conv) -> bool:
    return (isinstance(conv, nn.Conv3d) and conv.kernel_size == (1, 1, 1) and conv.stride == (1, 1, 1) and conv.padding == (0, 0, 0)
            and conv.dilation == (1, 1, 1) and conv.groups == 1 and conv.bias is None)


def block_pixels(block) -> Optional[int]:
    """X*Y of the maps the block is built for (its pyramid pooling's kernel covers the whole map), or None if it has none."""
    pp = getattr(block, "pyramid_pooling", None) if getattr(block, "use_pyramid_pooling", False) else None
    if pp is None:
        return None
    k = _triple(pp.features[0].avgpool.kernel_size)
    return int(k[1]) * int(k[2])


def block_reason(block) -> Optional[str]:
    """None if ``block`` (a reference TemporalBlock) is covered by the kernels, else the reason."""
    try:
        paths = block.convolution_paths
        convs = [paths[0][0].conv, paths[1][0].conv, paths[2].conv]
        if block.projection is not None:
            convs.append(block.projection[0])
    except (AttributeError, IndexError, TypeError):
        return f"{type(block).__name__} does not have the TemporalBlock structure"
    for c in convs:
        if not _is_1x1x1(c):
            return f"{c} is not a bias-free 1x1x1 Conv3d"
    if len({c.in_channels for c in convs}) != 1:
        return "the 1x1x1 convolutions take different inputs"
    return unsupported_reason(convs[0].in_channels, [c.out_channels for c in convs], 0, block_pixels(block))


class TensorCoreTemporalBlock(nn.Module):
    """Drop-in for a reference ``TemporalBlock`` whose four 1x1x1 input convolutions run as one tensor-core GEMM
    (``torch.ops.fiery_b200.temporal_entry``).  It holds the reference block's children under the same names (``state_dict`` keys
    are unchanged) and looks them up at call time, so ``SyncBatchNorm.convert_sync_batchnorm`` works before or after the swap.  The
    norms, activations, causal convolutions, pyramid pooling, aggregation and projection BN are the block's own modules; each norm
    and its ReLU, and the last one with the skip add, go through ``batch_norm.norm_act``."""

    def __init__(self, block):
        super().__init__()
        for name in ("in_channels", "half_channels", "out_channels", "kernels", "use_pyramid_pooling"):
            setattr(self, name, getattr(block, name))
        self.convolution_paths = block.convolution_paths
        if block.use_pyramid_pooling:
            self.pyramid_pooling = block.pyramid_pooling
        self.aggregation = block.aggregation
        self.projection = block.projection

    @classmethod
    def from_block(cls, block) -> "TensorCoreTemporalBlock":
        reason = block_reason(block)
        if reason is not None:
            raise ValueError(f"TemporalBlock not covered by the tensor-core kernels: {reason}")
        return cls(block)

    def _entry_convs(self):
        p = self.convolution_paths
        convs = [p[0][0].conv, p[1][0].conv, p[2].conv]
        return convs + [self.projection[0]] if self.projection is not None else convs

    def _tail(self, x: torch.Tensor, ys: Sequence[torch.Tensor], pooled: Optional[torch.Tensor],
              vector: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Everything after the four convolutions (temporal.py:268-281); ``x`` is the block input the skip adds when there is no
        projection.  ``pooled``: the pyramid pooling's broadcast, concatenated to the paths; ``vector``: instead, its (b, R, s) pooled
        vector, which ``temporal_aggregation`` takes without a concat."""
        p = self.convolution_paths
        paths = []
        for i in range(3):
            entry = p[i][0] if i < 2 else p[i]
            y = norm_act(entry.norm, entry.activation, ys[i])
            paths.append(p[i][1](y) if i < 2 else y)
        skip = self.projection[1](ys[3]) if self.projection is not None else x
        agg = self.aggregation[0]
        if vector is not None:
            z = torch.ops.fiery_b200.temporal_aggregation(paths, agg.conv.weight, vector)
        else:
            z = torch.cat(paths, dim=1)
            if pooled is not None:
                z = torch.cat([z, pooled], dim=1)
            z = agg.conv(z)
        # skip + relu(bn(z)): with a FusedBatchNorm3d, one apply that adds the skip
        return norm_act(agg.norm, agg.activation, z, residual=skip)

    def _folds_pooling(self, h: int, w: int) -> bool:
        """The pyramid pooling is the swapped module, its kernel covers this map and the aggregation kernel takes it: the block runs
        the pooled vector through ``temporal_aggregation``.  A covered aggregation on an X*Y the kernel does not take warns once."""
        pp = getattr(self, "pyramid_pooling", None)
        if not (self.use_pyramid_pooling and isinstance(pp, TensorCorePyramidPooling) and pp.covers(h, w)):
            return False
        if aggregation_block_reason(self) is not None:
            return False
        if (h * w) % 4:
            warn_once(("aggregation", h * w), f"fiery_b200: TemporalBlock aggregation on X*Y = {h * w} pixels is not covered by the "
                      "tensor-core kernel (it needs a multiple of 4); it runs as the reference's concat and Conv3d")
            return False
        return True

    def forward(self, *inputs):
        (x,) = inputs
        convs = self._entry_convs()
        pixels = x.shape[3] * x.shape[4]
        if pixels % 4:
            # only a block without pyramid pooling reaches this: install() checks the map size through its pooling kernel
            warn_once(("entry_pixels", pixels), f"fiery_b200: TemporalBlock input of X*Y = {pixels} pixels is not covered by the "
                      "tensor-core kernels (they need a multiple of 4); its 1x1x1 convolutions run as the reference's Conv3d")
            ys = [c(x) for c in convs]
        else:
            ys = torch.ops.fiery_b200.temporal_entry(x, [c.weight for c in convs], None)
        if self._folds_pooling(x.shape[3], x.shape[4]):
            return self._tail(x, ys, None, self.pyramid_pooling.vector(spatial_means(x)))
        pooled = self.pyramid_pooling(x) if self.use_pyramid_pooling else None
        return self._tail(x, ys, pooled)

    def forward_folded(self, x: torch.Tensor, extra: torch.Tensor) -> torch.Tensor:
        """The block on the input ``cat([x, extra broadcast over the map], channel)`` without building it: x (b, K, s, X, Y), extra
        (b, s, E) constant per frame (the egopose).  The block must have no skip without projection (its input is the concat)."""
        if self.projection is None:
            raise ValueError("the folded form needs a block with a projection: the skip would add the concatenated input")
        ys = torch.ops.fiery_b200.temporal_entry(x, [c.weight for c in self._entry_convs()], extra)
        if not self.use_pyramid_pooling:
            return self._tail(x, ys, None)
        h, w = x.shape[3], x.shape[4]
        pp = self.pyramid_pooling
        k = _uncovered_kernel(pp.features, h, w)
        if k is not None:
            raise ValueError(f"pyramid pooling kernel {k} does not cover the {h}x{w} map; the folded form needs one that does")
        # the swapped pooling's means come from the spatial-sums kernel, as in its unfolded forward; the reference pooling's from torch
        swapped = isinstance(pp, TensorCorePyramidPooling)
        means = spatial_means(x) if swapped else x.float().mean(dim=(3, 4))
        vector = pyramid_vector(pp.features, torch.cat([means, extra.float().permute(0, 2, 1)], dim=1))
        if swapped and self._folds_pooling(h, w):
            return self._tail(x, ys, None, vector)
        return self._tail(x, ys, vector[..., None, None].expand(*vector.shape, h, w))


def spatial_means(x: torch.Tensor) -> torch.Tensor:
    """(b, C, s, X, Y) -> (b, C, s) fp32 means over each pixel plane (``torch.ops.fiery_b200.spatial_sums`` / X*Y)."""
    return torch.ops.fiery_b200.spatial_sums(x) / (x.shape[3] * x.shape[4])


def _triple(v) -> Tuple[int, int, int]:
    """An ``AvgPool3d`` size as given (an int or a sequence) -> its (t, X, Y) tuple."""
    return tuple(v) if isinstance(v, (tuple, list)) else (v,) * 3


def _uncovered_kernel(features, h: int, w: int) -> Optional[Tuple[int, int, int]]:
    """The kernel of the first pool in ``features`` that does not span the whole h x w map, or None if every pool does."""
    return next((k for k in (_triple(f.avgpool.kernel_size) for f in features) if k[1:] != (h, w)), None)


def pyramid_vector(features, means: torch.Tensor) -> torch.Tensor:
    """The pyramid pooling of pools that each span the whole map, as the (b, R, s) vector of its values per frame, from the input's
    spatial means (b, C, s).  The 2-frame window averages frames t - 1 and t, and frame 0 alone (the pad is not counted); each pool's
    own ``conv_bn_relu`` runs on the (b, C, s + 1, 1, 1) window, whose extra last step (frame s - 1 alone) goes through BN with the
    others and is then dropped; the pools' outputs are concatenated over channels.  The bilinear upsampling of a 1x1 map that the
    reference applies next is a broadcast of this vector."""
    window = torch.cat([means[..., :1], (means[..., :-1] + means[..., 1:]) / 2, means[..., -1:]], dim=2)[..., None, None]
    return torch.cat([f.conv_bn_relu(window)[:, :, :-1, 0, 0] for f in features], 1)


def pooling_reason(pp) -> Optional[str]:
    """None if ``pp`` (a reference PyramidSpatioTemporalPooling) is one pool of the reference's (2, X, Y) window -- 2 frames, one
    frame of padding in front that is not counted, stride (1, X, Y) -- that ``TensorCorePyramidPooling`` computes from spatial means,
    else the reason.  Whether X x Y covers the map is checked at call time."""
    feats = getattr(pp, "features", None)
    if feats is None:
        return f"{type(pp).__name__} does not have the PyramidSpatioTemporalPooling structure"
    if len(feats) != 1:
        return f"{len(feats)} pool sizes (the swap covers one pool over the whole map)"
    ap = getattr(feats[0], "avgpool", None)
    if not isinstance(ap, nn.AvgPool3d) or not hasattr(feats[0], "conv_bn_relu"):
        return f"{feats[0]} is not an AvgPool3d followed by conv_bn_relu"
    k, stride, padding = _triple(ap.kernel_size), _triple(ap.stride), _triple(ap.padding)
    if (k[0] != 2 or stride != (1, k[1], k[2]) or padding != (1, 0, 0) or ap.count_include_pad or ap.ceil_mode
            or ap.divisor_override is not None):
        return f"pool {ap} is not the (2, X, Y) window with stride (1, X, Y) and one uncounted frame of padding"
    return None


def aggregation_block_reason(block) -> Optional[str]:
    """None if ``block``'s aggregation conv (bias-free 1x1x1 over the three paths and the pooled channels) is covered by the
    aggregation kernel, else the reason.  X*Y is checked at call time."""
    try:
        agg = block.aggregation[0]
        conv, _, _ = agg.conv, agg.norm, agg.activation
        seg = [int(block.half_channels)] * len(block.convolution_paths)
    except (AttributeError, IndexError, TypeError):
        return f"{type(block).__name__} does not have the TemporalBlock aggregation structure"
    if not _is_1x1x1(conv):
        return f"aggregation {conv} is not a bias-free 1x1x1 Conv3d"
    if conv.in_channels <= sum(seg):
        return f"aggregation takes {conv.in_channels} channels: no pooled channels after the paths' {sum(seg)}"
    return aggregation_reason(conv.out_channels, seg)


class TensorCorePyramidPooling(nn.Module):
    """Drop-in for a reference ``PyramidSpatioTemporalPooling`` with one pool over the whole map (the one ``TemporalModel`` builds,
    fiery/models/temporal_model.py:23).  It holds the reference module's ``features`` (``state_dict`` keys unchanged) and computes the
    pool from the input's spatial means (``torch.ops.fiery_b200.spatial_sums``): the 2-frame window over the means, then the
    reference's own ``conv_bn_relu`` on (b, C, s + 1, 1, 1), the padded last frame dropped after BN.  ``forward`` returns the
    broadcast over the map as an expanded (stride-0) view; the bilinear upsampling of a 1x1 map it replaces is that broadcast, and
    its adjoint a spatial sum.  Inside a ``TensorCoreTemporalBlock`` the block takes ``vector`` instead and never builds the broadcast.
    A map its pool does not cover runs the reference's computation, with one warning."""

    def __init__(self, pp):
        super().__init__()
        self.features = pp.features

    @classmethod
    def from_module(cls, pp) -> "TensorCorePyramidPooling":
        reason = pooling_reason(pp)
        if reason is not None:
            raise ValueError(f"PyramidSpatioTemporalPooling not covered by the spatial-sums pooling: {reason}")
        return cls(pp)

    def covers(self, h: int, w: int) -> bool:
        return _uncovered_kernel(self.features, h, w) is None

    def vector(self, means: torch.Tensor) -> torch.Tensor:
        """(b, C, s) spatial means -> the (b, R, s) pooled vector (``pyramid_vector``)."""
        return pyramid_vector(self.features, means)

    def forward(self, *inputs):
        (x,) = inputs
        b, _, s, h, w = x.shape
        if not self.covers(h, w):
            warn_once(("pooling", h, w), f"fiery_b200: pyramid pooling {_triple(self.features[0].avgpool.kernel_size)} does not cover "
                      f"the {h}x{w} map; it runs as the reference's average pool and bilinear upsampling")
            out = []
            for f in self.features:
                y = f(x)[:, :, :-1].contiguous()
                c = y.shape[1]
                y = F.interpolate(y.reshape(b * s, c, *y.shape[-2:]), (h, w), mode="bilinear", align_corners=False)
                out.append(y.reshape(b, c, s, h, w))
            return torch.cat(out, 1)
        v = self.vector(spatial_means(x))
        return v[..., None, None].expand(*v.shape, h, w)


def temporal_model_forward(temporal_model, bev: torch.Tensor, future_egomotion: torch.Tensor) -> torch.Tensor:
    """fiery.py:148-158 (egopose concat + ``self.temporal_model(x)``) without the concat: bev (b, s, C, X, Y) the warped BEV,
    future_egomotion (b, s, E).  The egopose fed at frame t is zeros at t = 0 and ``future_egomotion[:, t - 1]`` after that, as in the
    reference.  The first block must be a ``TensorCoreTemporalBlock`` (``install.use_tensor_core_temporal_model``)."""
    blocks = temporal_model.model
    first = blocks[0]
    if not isinstance(first, TensorCoreTemporalBlock):
        raise TypeError("temporal_model_forward needs the first block swapped: call install.use_tensor_core_temporal_model(model)")
    b, s = bev.shape[:2]
    extra = torch.cat([torch.zeros_like(future_egomotion[:, :1]), future_egomotion[:, :s - 1]], dim=1)
    x = first.forward_folded(bev.permute(0, 2, 1, 3, 4), extra)
    for m in list(blocks)[1:]:
        x = m(x)
    x = x.permute(0, 2, 1, 3, 4).contiguous()
    return x[:, (temporal_model.receptive_field - 1):]
