"""ctypes binding of libfiery_b200.so (C ABI: include/fiery_b200.h), the one helper every launch goes through (``call``), the
cache of the tensor-core layers' weight packs (``packed``), and the host rules the operators share: input layouts, workspaces and
the once-only warnings of every swap and fallback (``warn_once``).

There is no fallback: if the shared library is missing or a call fails this module raises.  Build it in-tree with
``python -m fiery_b200.build`` (the built ``.so`` travels with the repo snapshot to the GPU box).
"""
from __future__ import annotations

import collections
import ctypes
import os
import warnings
from ctypes import POINTER, c_char_p, c_double, c_float, c_int32, c_int64, c_size_t, c_uint8, c_void_p

import torch

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libfiery_b200.so")
ABI_VERSION = 2

DTYPE_F32, DTYPE_F16 = 0, 1
CALIB_RAW, CALIB_COMPOSED = 0, 1
BEV_NCHW, BEV_NHWC = 0, 1


class FieryError(RuntimeError):
    """A fiery_b200 C-ABI call returned a negative status."""


class LiftDesc(ctypes.Structure):
    """Mirror of ``fiery_lift_desc_t``."""

    _fields_ = [
        ("n_frames", c_int32), ("n_cameras", c_int32), ("depth_bins", c_int32), ("channels", c_int32),
        ("feat_h", c_int32), ("feat_w", c_int32),
        ("bev_x", c_int32), ("bev_y", c_int32), ("bev_z", c_int32),
        ("bev_offset", c_float * 3), ("bev_resolution", c_float * 3),
        ("z_valid_lo", c_float), ("z_valid_hi", c_float),
        ("use_depth_distribution", c_int32), ("head_dtype", c_int32), ("calib_mode", c_int32), ("bev_layout", c_int32),
    ]


class TemporalEntryDesc(ctypes.Structure):
    """Mirror of ``fiery_temporal_entry_desc_t``."""

    _fields_ = [
        ("batch", c_int32), ("frames", c_int32), ("pixels", c_int32), ("in_channels", c_int32), ("extra_channels", c_int32),
        ("n_segments", c_int32), ("seg_channels", c_int32 * 4),
        ("in_stride_b", c_int64), ("in_stride_t", c_int64), ("in_stride_c", c_int64),
    ]


class SpatialSumsDesc(ctypes.Structure):
    """Mirror of ``fiery_spatial_sums_desc_t``."""

    _fields_ = [
        ("batch", c_int32), ("channels", c_int32), ("frames", c_int32), ("pixels", c_int32),
        ("stride_b", c_int64), ("stride_c", c_int64), ("stride_t", c_int64),
    ]


class CausalConv3dDesc(ctypes.Structure):
    """Mirror of ``fiery_causal_conv3d_desc_t``."""

    _fields_ = [
        ("batch", c_int32), ("frames", c_int32), ("grid_x", c_int32), ("grid_y", c_int32), ("in_channels", c_int32),
        ("out_channels", c_int32), ("kt", c_int32),
    ]


class BatchNormDesc(ctypes.Structure):
    """Mirror of ``fiery_batch_norm_desc_t``."""

    _fields_ = [
        ("batch", c_int32), ("channels", c_int32), ("frames", c_int32), ("pixels", c_int32),
        ("stride_b", c_int64), ("stride_c", c_int64), ("stride_t", c_int64),
        ("training", c_int32), ("relu", c_int32), ("eps", c_double),
    ]


class SpatialGruDesc(ctypes.Structure):
    """Mirror of ``fiery_spatial_gru_desc_t``."""

    _fields_ = [
        ("batch", c_int32), ("frames", c_int32), ("x_frames", c_int32), ("grid_x", c_int32), ("grid_y", c_int32),
        ("x_channels", c_int32), ("h_channels", c_int32),
        ("x_stride_b", c_int64), ("x_stride_t", c_int64), ("x_stride_c", c_int64),
        ("training", c_int32), ("eps", c_double), ("bias_init", c_float),
    ]


class Conv3x3Desc(ctypes.Structure):
    """Mirror of ``fiery_conv3x3_desc_t``."""

    _fields_ = [("maps", c_int32), ("grid_x", c_int32), ("grid_y", c_int32), ("in_channels", c_int32 * 2), ("out_channels", c_int32 * 2)]


class BottleneckDesc(ctypes.Structure):
    """Mirror of ``fiery_bottleneck_desc_t``."""

    _fields_ = [("maps", c_int32), ("grid_x", c_int32), ("grid_y", c_int32), ("channels", c_int32), ("training", c_int32),
                ("eps", c_double)]


class OutputHeadDesc(ctypes.Structure):
    """Mirror of ``fiery_output_head_desc_t``."""

    _fields_ = [("maps", c_int32), ("grid_x", c_int32), ("grid_y", c_int32), ("channels", c_int32), ("n_out", c_int32),
                ("training", c_int32), ("eps", c_double)]


# name -> (restype, argtypes); every symbol include/fiery_b200.h declares
SIGNATURES = {
    "fiery_abi_version": (c_int32, []),
    "fiery_last_error": (c_char_p, []),
    "fiery_lift_plan_bytes": (c_size_t, [POINTER(LiftDesc)]),
    "fiery_lift_plan": (c_int32, [POINTER(LiftDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_lift_scratch_bytes": (c_size_t, [POINTER(LiftDesc)]),
    "fiery_lift_forward_launches": (c_int32, [POINTER(LiftDesc)]),
    "fiery_lift_forward": (c_int32, [POINTER(LiftDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_lift_forward_warped": (c_int32, [POINTER(LiftDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_lift_forward_timed": (c_int32, [POINTER(LiftDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_int32, POINTER(c_float), POINTER(c_int32),
                                           POINTER(c_int32)]),
    "fiery_lift_deterministic_workspace_bytes": (c_size_t, [POINTER(LiftDesc)]),
    "fiery_lift_forward_deterministic": (c_int32, [POINTER(LiftDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                   c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_lift_set_max_chunk_frames": (None, [c_int32]),
    "fiery_lift_workspace_bytes": (c_size_t, [POINTER(LiftDesc)]),
    "fiery_lift_backward": (c_int32, [POINTER(LiftDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_lift_point_indices": (c_int32, [POINTER(LiftDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_compose_calibration": (c_int32, [c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_voxels_summing_plan": (c_int32, [c_int64, c_void_p, c_void_p, POINTER(c_int64), c_void_p]),
    "fiery_voxels_summing_forward": (c_int32, [c_int64, c_int32, c_int64, c_void_p, c_void_p, c_void_p, c_int64,
                                               c_void_p, c_void_p, c_void_p]),
    "fiery_voxels_summing_backward": (c_int32, [c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_voxels_summing_deterministic_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "fiery_voxels_summing_forward_deterministic": (c_int32, [c_int64, c_int32, c_int64, c_void_p, c_void_p, c_void_p, c_int64,
                                                             c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_depth_layer_forward": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_bev_conv_pack_weights": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "fiery_bev_first_conv_forward": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p]),
    "fiery_bev_conv_pack_weights_transposed": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "fiery_bev_first_conv_backward_data": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_bev_first_conv_backward_weight_workspace_bytes": (c_size_t, [c_int32, c_int32, c_int32]),
    "fiery_bev_first_conv_backward_weight": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_temporal_entry_packed_bytes": (c_size_t, [POINTER(TemporalEntryDesc)]),
    "fiery_temporal_entry_pack_weights": (c_int32, [POINTER(TemporalEntryDesc), c_void_p, c_void_p, c_void_p]),
    "fiery_temporal_entry_forward": (c_int32, [POINTER(TemporalEntryDesc), c_void_p, c_void_p, c_void_p, POINTER(c_void_p), c_void_p]),
    "fiery_temporal_entry_backward_data": (c_int32, [POINTER(TemporalEntryDesc), POINTER(c_void_p), c_void_p, c_void_p, c_void_p]),
    "fiery_temporal_entry_backward_weight_workspace_bytes": (c_size_t, [POINTER(TemporalEntryDesc)]),
    "fiery_temporal_entry_backward_weight": (c_int32, [POINTER(TemporalEntryDesc), c_void_p, c_void_p, POINTER(c_void_p), c_void_p,
                                                       c_void_p, c_void_p]),
    "fiery_temporal_aggregation_forward": (c_int32, [POINTER(TemporalEntryDesc), POINTER(c_void_p), c_void_p, c_void_p, c_void_p,
                                                     c_void_p]),
    "fiery_spatial_sums": (c_int32, [POINTER(SpatialSumsDesc), c_void_p, c_void_p, c_void_p]),
    "fiery_causal_conv3d_packed_bytes": (c_size_t, [POINTER(CausalConv3dDesc)]),
    "fiery_causal_conv3d_pack_weights": (c_int32, [POINTER(CausalConv3dDesc), c_void_p, c_void_p, c_void_p]),
    "fiery_causal_conv3d_forward": (c_int32, [POINTER(CausalConv3dDesc), c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_causal_conv3d_backward_data": (c_int32, [POINTER(CausalConv3dDesc), c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_causal_conv3d_backward_weight_workspace_bytes": (c_size_t, [POINTER(CausalConv3dDesc)]),
    "fiery_causal_conv3d_backward_weight": (c_int32, [POINTER(CausalConv3dDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_batch_norm_workspace_bytes": (c_size_t, [POINTER(BatchNormDesc)]),
    "fiery_batch_norm_forward": (c_int32, [POINTER(BatchNormDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_batch_norm_backward": (c_int32, [POINTER(BatchNormDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_batch_norm_sync_workspace_bytes": (c_size_t, [POINTER(BatchNormDesc)]),
    "fiery_batch_norm_local_stats": (c_int32, [POINTER(BatchNormDesc)] + [c_void_p] * 4),
    "fiery_batch_norm_forward_gathered": (c_int32, [POINTER(BatchNormDesc), c_int32] + [c_void_p] * 11),
    "fiery_batch_norm_local_grad_sums": (c_int32, [POINTER(BatchNormDesc)] + [c_void_p] * 11),
    "fiery_batch_norm_backward_gathered": (c_int32, [POINTER(BatchNormDesc), c_int32] + [c_void_p] * 10),
    "fiery_spatial_gru_forward_step_begin": (c_int32, [POINTER(SpatialGruDesc), c_int32] + [c_void_p] * 9),
    "fiery_spatial_gru_forward_step_end": (c_int32, [POINTER(SpatialGruDesc), c_int32, c_int32] + [c_void_p] * 11),
    "fiery_spatial_gru_backward_step_begin": (c_int32, [POINTER(SpatialGruDesc), c_int32] + [c_void_p] * 13),
    "fiery_spatial_gru_backward_step_end": (c_int32, [POINTER(SpatialGruDesc), c_int32, c_int32] + [c_void_p] * 13),
    "fiery_spatial_gru_backward_weights": (c_int32, [POINTER(SpatialGruDesc)] + [c_void_p] * 12),
    "fiery_spatial_gru_packed_bytes": (c_size_t, [POINTER(SpatialGruDesc)]),
    "fiery_spatial_gru_pack_weights": (c_int32, [POINTER(SpatialGruDesc), c_void_p, c_void_p, c_void_p, c_void_p]),
    "fiery_spatial_gru_saved_bytes": (c_size_t, [POINTER(SpatialGruDesc)]),
    "fiery_spatial_gru_forward_workspace_bytes": (c_size_t, [POINTER(SpatialGruDesc)]),
    "fiery_spatial_gru_forward": (c_int32, [POINTER(SpatialGruDesc)] + [c_void_p] * 14),
    "fiery_spatial_gru_backward_workspace_bytes": (c_size_t, [POINTER(SpatialGruDesc)]),
    "fiery_spatial_gru_backward": (c_int32, [POINTER(SpatialGruDesc)] + [c_void_p] * 19),
    "fiery_conv3x3_packed_bytes": (c_size_t, [POINTER(Conv3x3Desc)]),
    "fiery_conv3x3_pack_weights": (c_int32, [POINTER(Conv3x3Desc), c_void_p, c_void_p, c_void_p]),
    "fiery_conv3x3_forward": (c_int32, [POINTER(Conv3x3Desc)] + [c_void_p] * 6),
    "fiery_conv3x3_backward_data": (c_int32, [POINTER(Conv3x3Desc)] + [c_void_p] * 6),
    "fiery_conv3x3_backward_weight_workspace_bytes": (c_size_t, [POINTER(Conv3x3Desc)]),
    "fiery_conv3x3_backward_weight": (c_int32, [POINTER(Conv3x3Desc)] + [c_void_p] * 6),
    "fiery_bottleneck_packed_bytes": (c_size_t, [POINTER(BottleneckDesc)]),
    "fiery_bottleneck_pack_weights": (c_int32, [POINTER(BottleneckDesc)] + [c_void_p] * 5),
    "fiery_bottleneck_forward_workspace_bytes": (c_size_t, [POINTER(BottleneckDesc)]),
    "fiery_bottleneck_forward": (c_int32, [POINTER(BottleneckDesc), c_void_p, c_void_p, POINTER(c_void_p)] + [c_void_p] * 7),
    "fiery_bottleneck_backward_workspace_bytes": (c_size_t, [POINTER(BottleneckDesc)]),
    "fiery_bottleneck_backward": (c_int32, [POINTER(BottleneckDesc)] + [c_void_p] * 7 + [POINTER(c_void_p)] + [c_void_p] * 4
                                  + [POINTER(c_void_p), c_void_p, c_void_p]),
    "fiery_bottleneck_sync_forward_stage": (c_int32, [POINTER(BottleneckDesc), c_int32, c_int32] + [c_void_p] * 3 + [POINTER(c_void_p)]
                                            + [c_void_p] * 9),
    "fiery_bottleneck_sync_backward_stage": (c_int32, [POINTER(BottleneckDesc), c_int32, c_int32] + [c_void_p] * 8 + [POINTER(c_void_p)]
                                             + [c_void_p] * 4 + [POINTER(c_void_p)] + [c_void_p] * 3),
    "fiery_output_head_packed_bytes": (c_size_t, [POINTER(OutputHeadDesc)]),
    "fiery_output_head_pack_weights": (c_int32, [POINTER(OutputHeadDesc)] + [c_void_p] * 3),
    "fiery_output_head_forward_workspace_bytes": (c_size_t, [POINTER(OutputHeadDesc)]),
    "fiery_output_head_forward": (c_int32, [POINTER(OutputHeadDesc)] + [c_void_p] * 11),
    "fiery_output_head_backward_workspace_bytes": (c_size_t, [POINTER(OutputHeadDesc)]),
    "fiery_output_head_backward": (c_int32, [POINTER(OutputHeadDesc)] + [c_void_p] * 14),
    "fiery_warp_theta": (c_int32, [c_int32, c_int32, c_int32, c_void_p, c_float, c_float, c_void_p, c_void_p, c_void_p]),
    "fiery_warp_features_forward": (c_int32, [c_int32, c_int32, c_int32, c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                                              c_int64, c_int32, c_void_p]),
    "fiery_warp_features_backward": (c_int32, [c_int32, c_int32, c_int32, c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                                               c_int64, c_int32, c_void_p]),
}

_lib = None


def load() -> ctypes.CDLL:
    """Loads the shared library once; raises ``FieryError`` if it is absent or has the wrong ABI."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FieryError(f"{LIB_PATH} not found: build it with `python -m fiery_b200.build` "
                         "(fiery_b200 has no CPU fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing
        fn.restype = restype
        fn.argtypes = argtypes
    got = lib.fiery_abi_version()
    if got != ABI_VERSION:
        raise FieryError(f"libfiery_b200.so has ABI version {got}, this package expects {ABI_VERSION}: rebuild")
    _lib = lib
    return lib


def check(status: int, what: str) -> None:
    if status != 0:
        msg = load().fiery_last_error()
        raise FieryError(f"{what} failed ({status}): {msg.decode() if msg else 'no message'}")


@torch.compiler.disable          # the raw handle exists on eager streams only: a C-ABI call breaks a torch.compile graph here
def _stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _require_cuda(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise FieryError(f"{name} must be a CUDA tensor: fiery_b200 has no CPU path (got device {t.device})")


def call(entry: str, device: torch.device, *args) -> None:
    """``lib.<entry>(*args, stream)`` with ``device`` current and its current stream as the last argument; raises ``FieryError``
    under the entry's name if the call fails."""
    with torch.cuda.device(device):
        check(getattr(load(), entry)(*args, _stream_ptr(device)), entry)


def f32(t: torch.Tensor) -> torch.Tensor:
    """A contiguous fp32 tensor: the layout the kernels read."""
    return t.float().contiguous() if t.dtype != torch.float32 else t.contiguous()


def f32_planes(x: torch.Tensor) -> torch.Tensor:
    """A (b, C, s, X, Y) tensor as the pixel-plane kernels read it: x itself when it is fp32 with contiguous pixel planes (any
    b / C / s strides), else a contiguous fp32 copy."""
    _, _, _, h, w = x.shape
    planes_contiguous = (x.stride(4) == 1 or w == 1) and (x.stride(3) == w or h == 1)
    return x if x.dtype == torch.float32 and planes_contiguous else f32(x)


def workspace(nbytes: int, device: torch.device) -> torch.Tensor:
    """A uint8 device workspace of ``nbytes`` bytes, never empty, so the kernels get a valid pointer even when they need none."""
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


_warned = set()


def warn_once(key, msg: str, stacklevel: int = 2) -> None:
    """``warnings.warn(msg, RuntimeWarning)`` the first time ``key`` is seen, until ``install.uninstall()`` forgets them all;
    ``stacklevel`` counts from the caller, as ``warnings.warn``'s does."""
    if key not in _warned:
        _warned.add(key)
        warnings.warn(msg, RuntimeWarning, stacklevel=stacklevel + 1)


# (pack function, args, device, the weights' data_ptrs) -> (the weights' versions, aliases of the weights, pack).  The aliases keep the
# weights' memory alive, so no other tensor can take an address in the cache while its entry exists; a weight's version counter
# (shared with its views, its aliases and the Parameter) changes with each in-place update, e.g. an optimizer step or a checkpoint
# load.  One training step of a model with every layer swapped uses one pack per DepthLayer operand dtype, two for FirstConv (the
# transposed one for the input gradient), four per TemporalBlock (its entry, two causal convolutions and its aggregation) and one per
# Bottleneck3D: 19 for the four temporal blocks of a 5-frame receptive field, and one per SpatialGRU and Bottleneck: 12 for a swapped
# FuturePrediction, and one per output head: 4 for a swapped Decoder.  The bound leaves room for in-between layers (up to four per block there) without a step ever evicting a pack it
# uses again.
_PACK_CACHE_SIZE = 48
_pack_cache: "collections.OrderedDict[tuple, tuple]" = collections.OrderedDict()


@torch.compiler.disable          # host bookkeeping on data_ptr and _version: runs eagerly, never compiled into a graph
def packed(pack, weights, *args):
    """``pack(weights, *args)``, made at most once per version of ``weights`` (a tensor or a list of tensors)."""
    ws = (weights,) if isinstance(weights, torch.Tensor) else tuple(weights)
    key = (pack, args, ws[0].device) + tuple(w.data_ptr() for w in ws)
    versions = tuple(w._version for w in ws)
    entry = _pack_cache.get(key)
    if entry is None or entry[0] != versions or any(a.shape != w.shape for a, w in zip(entry[1], ws)):
        entry = (versions, [w.detach() for w in ws], pack(weights, *args))
        _pack_cache[key] = entry
        while len(_pack_cache) > _PACK_CACHE_SIZE:
            _pack_cache.popitem(last=False)
    _pack_cache.move_to_end(key)
    return entry[2]
