"""Rebind the reference's call sites to the CUDA path (INTEGRATION.md).

``install()`` patches an importable ``fiery`` package (the unmodified reference) so that ``Fiery.forward``
(fiery/models/fiery.py:130-191) runs on the fused lift without any source change:

  * ``fiery.utils.geometry.VoxelsSumming`` and ``fiery.models.fiery.VoxelsSumming`` (the name is bound at import,
    fiery.py:10) -> ``fiery_b200.geometry.VoxelsSumming``                                   [level "voxels_summing"]
  * ``Fiery.calculate_birds_eye_view_features`` (fiery.py:275) -> ``fiery_b200.lift.calculate_birds_eye_view_features``
                                                                                             [level "fused", default]
  * ``fiery.models.fiery.cumulative_warp_features`` (bound at import, fiery.py:10; call site fiery.py:143) and
    ``fiery.utils.geometry.cumulative_warp_features`` / ``warp_features`` -> ``fiery_b200.warp``       [level "all"]
"""
from __future__ import annotations

import functools
import importlib

import torch

from ._lib import _warned, warn_once
from .geometry import VoxelsSumming
from .lift import calculate_birds_eye_view_features
from .warp import cumulative_warp_features, warp_features

_saved = {}


def unsupported_reason(model, x):
    """None if the fused kernels cover this model's lift configuration, else the reason (the limits of
    fiery_b200/csrc: include/fiery_b200.h).  CPU tensors are NOT a reason: there is no CPU path and the call raises."""
    h, w = x.shape[-2] // model.encoder_downsample, x.shape[-1] // model.encoder_downsample
    D = model.frustum.shape[0]
    if int(model.encoder_out_channels) != 64:
        return f"MODEL.ENCODER.OUT_CHANNELS={int(model.encoder_out_channels)} (kernels are built for 64)"
    if D > 48:
        return f"{D} depth bins (kernels are built for <= 48)"
    if h > 32 or w % 4:
        return f"feature map {h}x{w} (kernels need h <= 32 and w % 4 == 0)"
    if int(model.bev_dimension[2]) != 1:
        return "more than one height cell"
    return None


def _bev_features(self, x, intrinsics, extrinsics):
    """Installed as ``Fiery.calculate_birds_eye_view_features``: the fused lift where the kernels cover the configuration,
    the reference's own method (unpatched behaviour, its own device) where they do not."""
    reason = unsupported_reason(self, x)
    if reason is None:
        return calculate_birds_eye_view_features(self, x, intrinsics, extrinsics)
    warn_once(("bev", reason), f"fiery_b200: lift configuration not covered by the CUDA kernels ({reason}); "
                               "running the reference's own calculate_birds_eye_view_features")
    return _saved["bev"](self, x, intrinsics, extrinsics)


def _bilinear_only(ours, saved_key):
    """Feature warps (mode='bilinear', fiery.py:143) run on the CUDA kernel.  The trainer's label warps use mode='nearest'
    (trainer.py, cumulative_warp_features_reverse): sample positions agree with torch only to ~1e-4, which can flip a
    nearest-neighbour pick at a tie, so those stay on the reference's function."""
    @functools.wraps(ours)
    def fn(x, flow, mode="nearest", spatial_extent=None):
        if mode == "bilinear" or _saved.get(saved_key) is None:
            return ours(x, flow, mode=mode, spatial_extent=spatial_extent)
        return _saved[saved_key](x, flow, mode=mode, spatial_extent=spatial_extent)
    return fn


def install(level: str = "fused"):
    if level not in ("fused", "voxels_summing", "all"):
        raise ValueError("level must be 'fused', 'voxels_summing' or 'all'")
    geometry = importlib.import_module("fiery.utils.geometry")
    fiery_mod = importlib.import_module("fiery.models.fiery")
    if not _saved:
        _saved["VoxelsSumming"] = geometry.VoxelsSumming
        _saved["bev"] = fiery_mod.Fiery.calculate_birds_eye_view_features
        _saved["cwf"] = getattr(geometry, "cumulative_warp_features", None)
        _saved["wf"] = getattr(geometry, "warp_features", None)
        _saved["cwf_model"] = getattr(fiery_mod, "cumulative_warp_features", None)
    geometry.VoxelsSumming = VoxelsSumming
    fiery_mod.VoxelsSumming = VoxelsSumming
    if level in ("fused", "all"):
        fiery_mod.Fiery.calculate_birds_eye_view_features = _bev_features
    if level == "all":
        geometry.cumulative_warp_features = _bilinear_only(cumulative_warp_features, "cwf")
        geometry.warp_features = _bilinear_only(warp_features, "wf")
        fiery_mod.cumulative_warp_features = _bilinear_only(cumulative_warp_features, "cwf_model")
    return fiery_mod.Fiery


def use_tensor_core_depth_layer(model):
    """Replace ``model.encoder.depth_layer`` (``nn.Conv2d(128, D + C, 1)``, fiery/models/encoder.py:36) of a ``Fiery`` instance by
    ``fiery_b200.depth_layer.DepthLayer`` sharing the same Parameters (``state_dict`` keys unchanged): under autocast the backbone's
    half features go straight to an fp32 head tensor, the dtype the lift computes in.  Returns the model; layers the kernel does not
    cover (input channels != 128, more than 128 outputs) are left alone with one warning."""
    from .depth_layer import DepthLayer
    conv = model.encoder.depth_layer
    if isinstance(conv, DepthLayer):
        return model
    if conv.in_channels != 128 or conv.out_channels > 128 or conv.kernel_size != (1, 1):
        warn_once(("depth_layer", conv.in_channels, conv.out_channels),
                  f"fiery_b200: depth_layer {conv.in_channels}->{conv.out_channels} not covered by the tensor-core kernel; left as is")
        return model
    model.encoder.depth_layer = DepthLayer.from_conv(conv)
    return model


def use_tensor_core_first_conv(model):
    """Replace ``model.decoder.first_conv`` (``nn.Conv2d(64, 64, 7, stride=2, padding=3, bias=False)``, fiery/models/decoder.py:11) of
    a ``Fiery`` instance by ``fiery_b200.bev_conv.FirstConv(bn=None)`` sharing the same Parameter (``state_dict`` keys unchanged): the
    forward and both gradients run on the tensor-core kernels, on the channel-last layout the lift can emit.  ``bn1`` and ``relu``
    stay the reference's modules, so batch statistics train as before.  Returns the model; a second call does nothing, and a layer
    the kernels do not cover (e.g. ``in_channels != 64`` when EXTRA_IN_CHANNELS widens the temporal model) is left alone with one
    warning."""
    from .bev_conv import FirstConv
    conv = model.decoder.first_conv
    if isinstance(conv, FirstConv):
        return model
    covered = (isinstance(conv, torch.nn.Conv2d) and conv.in_channels == 64 and conv.out_channels == 64 and conv.kernel_size == (7, 7)
               and conv.stride == (2, 2) and conv.padding == (3, 3) and conv.dilation == (1, 1) and conv.groups == 1
               and conv.bias is None and conv.padding_mode == "zeros")
    if not covered:
        desc = (f"{conv.in_channels}->{conv.out_channels} k{conv.kernel_size} s{conv.stride}" if isinstance(conv, torch.nn.Conv2d)
                else type(conv).__name__)
        warn_once(("first_conv", desc), f"fiery_b200: first_conv {desc} not covered by the tensor-core kernels (they are built for "
                                        "Conv2d(64, 64, 7, stride=2, padding=3, bias=False)); left as is")
        return model
    model.decoder.first_conv = FirstConv.from_conv(conv)
    return model


_TEMPORAL_BLOCKS = ("TemporalBlock", "TensorCoreTemporalBlock")


def _blocks(blocks, *kinds):
    """(index, name, block) of each block in ``blocks`` whose class is named one of ``kinds``."""
    for i, (name, block) in enumerate(blocks._modules.items()):
        if type(block).__name__ in kinds:
            yield i, name, block


def _temporal_blocks(model):
    return getattr(model.temporal_model, "model", None)


def _swap(model, slots, swapped, reason, make, warning: str, entry: str = "{where}: {reason}", sep: str = "; ", root=_temporal_blocks):
    """Replace each module that ``slots(root(model))`` (by default ``model.temporal_model.model``) yields as ``(parent, name, module,
    where)`` by ``setattr(parent, name, make(module))``, unless it already is a ``swapped`` or ``reason(module)`` gives a reason to
    leave it.  A module reached under several names gets one replacement, set in each.  The modules left are listed, each as
    ``entry`` and ``sep``-separated, in one warning after ``warning``, given once per list.  Nothing happens when ``root`` finds
    nothing.  Returns the model."""
    blocks = root(model)
    if blocks is None:
        return model
    made, skipped = {}, []                      # made: id of a replaced module -> its replacement
    for parent, name, module, where in list(slots(blocks)):
        if isinstance(module, swapped):
            continue
        why = reason(module)
        if why is not None:
            skipped.append(entry.format(where=where, reason=why))
            continue
        if id(module) not in made:
            made[id(module)] = make(module)
        setattr(parent, name, made[id(module)])
    if skipped:
        warn_once((warning, tuple(skipped)), warning + sep.join(skipped), stacklevel=3)
    return model


def use_tensor_core_temporal_model(model):
    """Replace every covered ``TemporalBlock`` in ``model.temporal_model.model`` (fiery/models/temporal_model.py:27-45) of a ``Fiery``
    instance by ``fiery_b200.temporal.TensorCoreTemporalBlock``, which adopts the block's children (``state_dict`` keys unchanged) and
    runs its four 1x1x1 input convolutions as one tensor-core GEMM, forward and backward.  Returns the model; a second call does
    nothing.  A ``TemporalModelIdentity`` (the static configs) is left alone, and so are blocks the kernels do not cover (wrong
    kernel size or bias, shapes outside the limits, an X*Y the TMA cannot take), with one warning."""
    from .temporal import TensorCoreTemporalBlock, block_reason

    def slots(blocks):
        for i, name, block in _blocks(blocks, "TemporalBlock"):
            yield blocks, name, block, f"block {i}"
    return _swap(model, slots, TensorCoreTemporalBlock, block_reason, TensorCoreTemporalBlock,
                 "fiery_b200: TemporalBlock(s) not covered by the tensor-core kernels, left as is: ")


def use_tensor_core_causal_convs(model):
    """Replace every covered ``CausalConv3d`` under ``model.temporal_model.model`` of a ``Fiery`` instance -- ``convolution_paths[0][1]``
    and ``[1][1]`` of each ``TemporalBlock`` or ``TensorCoreTemporalBlock``, and ``layers.conv`` of each ``Bottleneck3D``
    (INBETWEEN_LAYERS > 0) -- by ``fiery_b200.causal_conv.TensorCoreCausalConv3d``, which adopts the module's children
    (``state_dict`` keys unchanged) and runs its pad and (kt, 3, 3) convolution on the tensor cores, forward and backward.  Works before
    or after ``use_tensor_core_temporal_model``.  Returns the model; a second call does nothing, and modules the kernels do not cover
    (more than 64 channels, another kernel size, a bias) are left alone with one warning."""
    from .causal_conv import TensorCoreCausalConv3d, module_reason

    def slots(blocks):
        for i, _, block in _blocks(blocks, *_TEMPORAL_BLOCKS, "Bottleneck3D"):
            if type(block).__name__ == "Bottleneck3D":
                yield block.layers, "conv", block.layers.conv, f"block {i} bottleneck"
            else:
                for p in (0, 1):
                    yield block.convolution_paths[p], "1", block.convolution_paths[p][1], f"block {i} path {p}"
    return _swap(model, slots, TensorCoreCausalConv3d, module_reason, TensorCoreCausalConv3d,
                 "fiery_b200: CausalConv3d module(s) not covered by the tensor-core kernels, left as is: ")


def use_tensor_core_pyramid_pooling(model):
    """Replace the ``pyramid_pooling`` (fiery/layers/temporal.py:167-215) of every ``TemporalBlock`` or ``TensorCoreTemporalBlock`` in
    ``model.temporal_model.model`` of a ``Fiery`` instance by ``fiery_b200.temporal.TensorCorePyramidPooling``, which adopts its
    ``features`` (``state_dict`` keys unchanged) and computes the pool from the input's spatial sums, with no average pool over the map
    and no bilinear upsampling.  In a ``TensorCoreTemporalBlock`` whose aggregation conv the kernel covers, the aggregation then runs
    as ``torch.ops.fiery_b200.temporal_aggregation``: no concat and no broadcast over the map.  Works before or after
    ``use_tensor_core_temporal_model`` and ``use_tensor_core_causal_convs``.  Returns the model; a second call does nothing, and a
    pooling that does not cover the whole map (several pool sizes, a kernel other than (2, X, Y)) is left alone with one warning."""
    from .temporal import TensorCorePyramidPooling, pooling_reason

    def slots(blocks):
        for i, _, block in _blocks(blocks, *_TEMPORAL_BLOCKS):
            if getattr(block, "use_pyramid_pooling", False):
                yield block, "pyramid_pooling", block.pyramid_pooling, f"block {i}"
    return _swap(model, slots, TensorCorePyramidPooling, pooling_reason, TensorCorePyramidPooling,
                 "fiery_b200: pyramid pooling(s) not covered by the spatial-sums kernel, left as is: ")


def use_fused_batch_norm(model):
    """Replace every module whose type is exactly ``nn.BatchNorm3d`` under ``model.temporal_model.model`` of a ``Fiery`` instance -- in
    reference blocks, swapped blocks and ``Bottleneck3D`` alike -- by ``fiery_b200.batch_norm.FusedBatchNorm3d``, which adopts its
    Parameters and buffers (``state_dict`` keys unchanged) and runs on the batch-norm kernels.  In a ``TensorCoreTemporalBlock`` and a
    ``TensorCoreCausalConv3d`` the ReLU after each norm, and the block's skip add, then run in the norm's apply pass.  The pyramid
    pooling's ``conv_bn_relu`` (a (b, R, s + 1, 1, 1) tensor) keeps its ``nn.BatchNorm3d``.  A ``SyncBatchNorm`` is left as it is, with
    one warning (``use_fused_sync_batch_norm`` swaps those); a ``FusedSyncBatchNorm`` is left as it is, silently.  Works before or
    after the other temporal swaps; a second call does nothing.  Returns the model."""
    from .batch_norm import FusedBatchNorm3d, FusedSyncBatchNorm

    def reason(norm):
        return "per-rank statistics" if isinstance(norm, torch.nn.SyncBatchNorm) else None
    # the warning's text gives the one reason, so it lists the skipped norms by name only; a FusedSyncBatchNorm is already swapped
    return _swap(model, _temporal_norms(torch.nn.BatchNorm3d, any_sync=True), (FusedBatchNorm3d, FusedSyncBatchNorm), reason,
                 FusedBatchNorm3d, "fiery_b200: SyncBatchNorm module(s) left as they are (use_fused_batch_norm computes per-rank "
                 "statistics only; use_fused_sync_batch_norm swaps them): ", entry="{where}", sep=", ")


def _temporal_norms(kind, any_sync: bool = False):
    """``_swap``'s slots for every module of type exactly ``kind`` (and, with ``any_sync``, every ``nn.SyncBatchNorm``) under the
    temporal model, but the pyramid pooling's."""
    def slots(blocks):
        for name, parent in blocks.named_modules():
            for key, child in parent.named_children():
                where = f"{name}.{key}" if name else key
                if "pyramid_pooling" not in where.split(".") and (type(child) is kind
                                                                  or (any_sync and isinstance(child, torch.nn.SyncBatchNorm))):
                    yield parent, key, child, where
    return slots


def use_fused_sync_batch_norm(model):
    """Replace every module of type exactly ``nn.SyncBatchNorm`` under ``model.temporal_model.model`` that ``use_fused_batch_norm``
    would swap were it a ``BatchNorm3d`` (the pyramid pooling's stays), and the ``conv_state_tilde.norm`` of every SpatialGRU in
    ``model.future_prediction.spatial_grus`` (the reference's or a ``TensorCoreSpatialGRU``), by
    ``fiery_b200.batch_norm.FusedSyncBatchNorm``.  It adopts the module's Parameters, buffers and ``process_group`` (``state_dict``
    keys unchanged) and gathers every rank's statistics and merges them on the kernels, as ``SyncBatchNorm`` would synchronize them;
    a swapped GRU then runs one gather per step each way.  Call it after ``SyncBatchNorm.convert_sync_batchnorm``; it works before or
    after the other temporal swaps and ``use_tensor_core_future_prediction`` (which then accepts the GRUs), and a second call does
    nothing.  Returns the model."""
    from .batch_norm import FusedSyncBatchNorm
    temporal = lambda m: _temporal_blocks(m) if hasattr(m, "temporal_model") else None      # noqa: E731  (a model may have none)
    _swap(model, _temporal_norms(torch.nn.SyncBatchNorm), FusedSyncBatchNorm, lambda m: None, FusedSyncBatchNorm, "", root=temporal)

    def gru_norms(grus):
        for i, (_, gru) in enumerate(grus._modules.items()):
            st = getattr(gru, "conv_state_tilde", None)
            norm = getattr(st, "norm", None) if st is not None else None
            if type(norm) is torch.nn.SyncBatchNorm:
                yield st, "norm", norm, f"spatial_grus[{i}]"
    return _swap(model, gru_norms, FusedSyncBatchNorm, lambda m: None, FusedSyncBatchNorm, "", root=_spatial_grus)


def _spatial_grus(model):
    fp = getattr(model, "future_prediction", None)
    return getattr(fp, "spatial_grus", None) if fp is not None else None


def use_tensor_core_future_prediction(model):
    """Replace every covered ``SpatialGRU`` in ``model.future_prediction.spatial_grus`` (fiery/models/future_prediction.py) of a
    ``Fiery`` instance by ``fiery_b200.future_prediction.TensorCoreSpatialGRU``, which adopts the module's convolutions and its
    ``ConvBlock`` (``state_dict`` keys unchanged) and runs all its steps as ``torch.ops.fiery_b200.spatial_gru``, forward and backward.
    Returns the model; a second call does nothing, a model without future prediction is returned untouched, and GRUs the kernels do
    not cover (another kernel size, a norm other than BatchNorm2d -- a SyncBatchNorm stays torch's --, an activation other than ReLU,
    more than 64 input or hidden channels) are left alone with one warning.  The ``Bottleneck``s stay as they are."""
    from .future_prediction import TensorCoreSpatialGRU, module_reason

    def slots(grus):
        for i, (name, gru) in enumerate(grus._modules.items()):
            yield grus, name, gru, f"spatial_grus[{i}]"
    return _swap(model, slots, TensorCoreSpatialGRU, module_reason, TensorCoreSpatialGRU.from_module,
                 "fiery_b200: SpatialGRU(s) not covered by the tensor-core kernels, left as is: ", root=_spatial_grus)


def _res_blocks(model):
    fp = getattr(model, "future_prediction", None)
    return getattr(fp, "res_blocks", None) if fp is not None else None


def use_tensor_core_bottlenecks(model):
    """Replace every covered ``Bottleneck`` in ``model.future_prediction.res_blocks`` (fiery/models/future_prediction.py) of a
    ``Fiery`` instance by ``fiery_b200.bottleneck.TensorCoreBottleneck``, which adopts the module's ``layers`` (``state_dict`` keys
    unchanged) and runs it as ``torch.ops.fiery_b200.bottleneck``: each inner BatchNorm2d and ReLU is applied as the next convolution
    reads its input, forward and backward.  Works before or after ``use_tensor_core_future_prediction``.  Returns the model; a second
    call does nothing, a model without future prediction is returned untouched, and Bottlenecks the kernels do not cover (a skip
    projection, another kernel size, dropout > 0, a norm other than BatchNorm2d -- a SyncBatchNorm stays torch's here;
    ``use_tensor_core_sync_bottlenecks`` swaps those --, more than 128 channels) are left alone with one warning."""
    from .bottleneck import TensorCoreBottleneck, module_reason

    def slots(res_blocks):
        for i, (_, stack) in enumerate(res_blocks._modules.items()):
            for name, block in stack._modules.items():
                yield stack, name, block, f"res_blocks[{i}][{name}]"
    return _swap(model, slots, TensorCoreBottleneck, module_reason, TensorCoreBottleneck.from_module,
                 "fiery_b200: Bottleneck(s) not covered by the tensor-core kernels, left as is: ", root=_res_blocks)


def use_tensor_core_sync_bottlenecks(model):
    """For every block in ``model.future_prediction.res_blocks`` of a ``Fiery`` instance (a reference ``Bottleneck`` or a
    ``TensorCoreBottleneck``) with a norm of type exactly ``nn.SyncBatchNorm``: when the kernels cover it with its three norms of that
    type, replace the three by ``fiery_b200.batch_norm.FusedSyncBatchNorm`` (same Parameters, buffers and ``process_group``;
    ``state_dict`` keys unchanged) and the block by a ``fiery_b200.bottleneck.TensorCoreBottleneck`` holding the same ``layers``.  In
    training over a group the block then runs ``SyncBottleneck``: the Bottleneck chain on the kernels with each norm's statistics
    gathered over the group, one gather per norm each way, as torch's converted modules.  Call it after
    ``SyncBatchNorm.convert_sync_batchnorm``; it works in any order with ``use_fused_sync_batch_norm``,
    ``use_tensor_core_future_prediction`` and ``use_tensor_core_bottlenecks``.  Returns the model; a second call does nothing, a model
    without future prediction is returned untouched, blocks without a SyncBatchNorm are left as they are, and converted blocks the
    kernels do not cover (a skip projection, dropout > 0, another kernel size, a mix of norm kinds) are left alone with one warning."""
    from .batch_norm import FusedSyncBatchNorm
    from .bottleneck import TensorCoreBottleneck, module_reason

    def slots(res_blocks):
        for i, (_, stack) in enumerate(res_blocks._modules.items()):
            for name, block in stack._modules.items():
                layers = getattr(block, "layers", None)
                norms = [m for m in layers.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)] if layers is not None else []
                if any(type(m) is torch.nn.SyncBatchNorm for m in norms):
                    yield stack, name, block, f"res_blocks[{i}][{name}]"

    def make(block):
        for abn in (block.layers.abn_down_project, block.layers.abn, block.layers.abn_up_project):
            abn[0] = FusedSyncBatchNorm(abn[0])
        return block if isinstance(block, TensorCoreBottleneck) else TensorCoreBottleneck(block)
    return _swap(model, slots, (), lambda block: module_reason(block, kinds=(torch.nn.SyncBatchNorm,)), make,
                 "fiery_b200: converted Bottleneck(s) not covered by the tensor-core kernels, left as is: ", root=_res_blocks)


def _decoder(model):
    return getattr(model, "decoder", None)


_OUTPUT_HEADS = ("segmentation_head", "instance_offset_head", "instance_center_head", "instance_future_head")


def use_tensor_core_output_heads(model):
    """Replace each covered output head of ``model.decoder`` (fiery/models/decoder.py:24-50: ``segmentation_head``,
    ``instance_offset_head``, ``instance_center_head`` and, when the model predicts future flow, ``instance_future_head``) of a ``Fiery``
    instance by ``fiery_b200.decoder.FusedOutputHead``, which adopts the head's children (``state_dict`` keys unchanged) and runs its
    BatchNorm2d, ReLU and 1x1 convolution as ``torch.ops.fiery_b200.output_head``, forward and backward; the 3x3 convolution stays
    cuDNN's.  Returns the model; a second call does nothing, a model without a decoder is returned untouched, and heads the kernels do
    not cover (a norm other than BatchNorm2d -- a SyncBatchNorm stays torch's --, more than 128 channels or 8 outputs, another
    structure) are left alone with one warning."""
    from .decoder import FusedOutputHead, module_reason

    def slots(decoder):
        for name in _OUTPUT_HEADS:
            head = getattr(decoder, name, None)
            if head is not None:
                yield decoder, name, head, name
    return _swap(model, slots, FusedOutputHead, module_reason, FusedOutputHead.from_module,
                 "fiery_b200: output head(s) not covered by the kernels, left as is: ", root=_decoder)


def uninstall():
    if not _saved:
        return
    geometry = importlib.import_module("fiery.utils.geometry")
    fiery_mod = importlib.import_module("fiery.models.fiery")
    geometry.VoxelsSumming = _saved["VoxelsSumming"]
    fiery_mod.VoxelsSumming = _saved["VoxelsSumming"]
    fiery_mod.Fiery.calculate_birds_eye_view_features = _saved["bev"]
    for mod, name, key in ((geometry, "cumulative_warp_features", "cwf"), (geometry, "warp_features", "wf"),
                           (fiery_mod, "cumulative_warp_features", "cwf_model")):
        if _saved.get(key) is not None:
            setattr(mod, name, _saved[key])
    _saved.clear()
    _warned.clear()
