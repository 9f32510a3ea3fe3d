"""Host-side constants of the lift and the ``VoxelsSumming`` drop-in.

Mirrors, with the same names, argument meaning and error behaviour:
  * ``calculate_birds_eye_view_parameters``  fiery/utils/geometry.py:39-58
  * ``Fiery.create_frustum``                 fiery/models/fiery.py:109-128
  * ``VoxelsSumming``                        fiery/utils/geometry.py:283-314  (call site fiery/models/fiery.py:261)
"""
from __future__ import annotations

import ctypes
from typing import Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import _require_cuda, _stream_ptr  # noqa: F401  (_stream_ptr: bench.py, tools/ and tests import it from here)


def calculate_birds_eye_view_parameters(x_bounds: Sequence[float], y_bounds: Sequence[float], z_bounds: Sequence[float]):
    """(bev_resolution f32[3], bev_start_position f32[3], bev_dimension i64[3]); fiery/utils/geometry.py:39-58."""
    rows = (x_bounds, y_bounds, z_bounds)
    bev_resolution = torch.tensor([float(r[2]) for r in rows])
    bev_start_position = torch.tensor([r[0] + r[2] / 2.0 for r in rows])
    bev_dimension = torch.tensor([(r[1] - r[0]) / r[2] for r in rows], dtype=torch.long)
    return bev_resolution, bev_start_position, bev_dimension


def create_frustum(final_dim: Tuple[int, int], encoder_downsample: int, d_bound: Sequence[float]) -> torch.Tensor:
    """(D, h, w, 3) grid of (pixel column, pixel row, depth); fiery/models/fiery.py:109-128."""
    H, W = final_dim
    fh, fw = H // encoder_downsample, W // encoder_downsample
    depth = torch.arange(*d_bound, dtype=torch.float)
    cols = torch.linspace(0, W - 1, fw, dtype=torch.float)
    rows = torch.linspace(0, H - 1, fh, dtype=torch.float)
    return torch.stack(torch.broadcast_tensors(cols.view(1, 1, fw), rows.view(1, fh, 1), depth.view(-1, 1, 1)), -1).contiguous()


def split_frustum(frustum: torch.Tensor):
    """The frustum is separable: column coordinate depends on w only, row on h, depth on D (fiery.py:115-127).
    Returns the three 1-D factors the kernels consume; raises if a (custom) frustum is not separable."""
    f = frustum.detach().float().cpu()
    if f.dim() != 4 or f.shape[-1] != 3:
        raise ValueError(f"frustum must be (D, h, w, 3), got {tuple(f.shape)}")
    u, v, d = f[0, 0, :, 0].clone(), f[0, :, 0, 1].clone(), f[:, 0, 0, 2].clone()
    ok = (torch.equal(f[..., 0], u.view(1, 1, -1).expand_as(f[..., 0]))
          and torch.equal(f[..., 1], v.view(1, -1, 1).expand_as(f[..., 1]))
          and torch.equal(f[..., 2], d.view(-1, 1, 1).expand_as(f[..., 2])))
    if not ok:
        raise ValueError("frustum is not separable into (column, row, depth) factors; only Fiery.create_frustum-style "
                         "frusta are supported")
    return u, v, d


def bev_offset_fp32(bev_start_position: torch.Tensor, bev_resolution: torch.Tensor) -> np.ndarray:
    """``bev_start_position - bev_resolution / 2.0`` evaluated in fp32 exactly as fiery/models/fiery.py:236 does."""
    return (bev_start_position.detach().float().cpu() - bev_resolution.detach().float().cpu() / 2.0).numpy().astype(np.float32)


def z_valid_interval(resolution_z: float, dim_z: int) -> Tuple[np.float32, np.float32]:
    """Closed fp32 interval [lo, hi] of a = z - offset_z with 0 <= trunc(fl(a / res_z)) < dim_z.

    a -> fl(a / res) is monotone, so the valid set is an interval of floats; its end points are found by stepping
    ulps around the analytic thresholds with IEEE division (numpy float32 == torch-CPU == __fdiv_rn)."""
    res = np.float32(resolution_z)
    q = lambda a: np.float32(a) / res                                    # noqa: E731
    lo = np.float32(-res)
    while q(lo) > np.float32(-1.0):
        lo = np.nextafter(lo, np.float32(-np.inf), dtype=np.float32)
    while not q(lo) > np.float32(-1.0):
        lo = np.nextafter(lo, np.float32(np.inf), dtype=np.float32)
    top = np.float32(dim_z)
    hi = np.float32(top * res)
    while q(hi) < top:
        hi = np.nextafter(hi, np.float32(np.inf), dtype=np.float32)
    while not q(hi) < top:
        hi = np.nextafter(hi, np.float32(-np.inf), dtype=np.float32)
    return np.float32(lo), np.float32(hi)


def _unfilled(shape, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
    """``torch.empty`` without the NaN fill ``torch.use_deterministic_algorithms(True)`` adds: for workspaces whose contents on entry
    do not matter and outputs the kernels overwrite completely (a fill of the lift's ~1 GB workspace would cost more than the lift)."""
    import torch.utils.deterministic as det
    old = det.fill_uninitialized_memory
    det.fill_uninitialized_memory = False
    try:
        return torch.empty(shape, dtype=dtype, device=device)
    finally:
        det.fill_uninitialized_memory = old


class VoxelsSumming(torch.autograd.Function):
    """Drop-in for ``fiery.utils.geometry.VoxelsSumming`` (geometry.py:283-314) on sm_90a.

    ``forward(ctx, x, geometry, ranks) -> (x_sum, geometry_kept)``: ``x`` (Nm, C) features and ``geometry`` (Nm, 3)
    int64 voxel coordinates, both ordered by ``ranks`` (Nm,) int64 ascending.  Returns the per-voxel sums (U, C) and
    the coordinates of the last row of every run (U, 3); ``geometry`` is marked non-differentiable (geometry.py:300).
    ``backward`` sends each voxel's gradient to all rows that were summed into it (geometry.py:305-314).
    The run sums are accumulated directly instead of via cumsum-and-subtract, so values agree with the reference to
    fp32 rounding (and are closer to the exact sum), not bit for bit.
    """

    @staticmethod
    def forward(ctx, x, geometry, ranks):
        _require_cuda(x, "x")
        lib = _lib.load()
        if x.dim() != 2 or geometry.dim() != 2 or geometry.shape[1] != 3 or ranks.dim() != 1:
            raise ValueError("expected x (Nm, C), geometry (Nm, 3), ranks (Nm,)")
        if not (x.shape[0] == geometry.shape[0] == ranks.shape[0]):
            raise ValueError("x, geometry and ranks disagree on the number of rows")
        n_rows, channels = x.shape
        xf = x if x.dtype == torch.float32 else x.float()
        if xf.stride(1) != 1:
            xf = xf.contiguous()
        coords = geometry.to(torch.int64).contiguous()
        rk = ranks.to(torch.int64).contiguous()
        dev = x.device
        seg = torch.empty(n_rows, dtype=torch.int32, device=dev)
        n_seg = ctypes.c_int64(0)
        _lib.call("fiery_voxels_summing_plan", dev, n_rows, rk.data_ptr(), seg.data_ptr(), ctypes.byref(n_seg))
        n_segments = int(n_seg.value)
        sums = torch.empty((n_segments, channels), dtype=torch.float32, device=dev)
        kept = torch.empty((n_segments, 3), dtype=torch.int64, device=dev)
        args = (n_rows, channels, xf.stride(0) if n_rows else channels, xf.data_ptr(), coords.data_ptr(), seg.data_ptr(),
                n_segments, sums.data_ptr(), kept.data_ptr())
        if torch.are_deterministic_algorithms_enabled():     # chunk-edge runs summed in chunk order instead of atomically
            ws = _unfilled(max(1, int(lib.fiery_voxels_summing_deterministic_workspace_bytes(n_rows, channels))), torch.uint8, dev)
            _lib.call("fiery_voxels_summing_forward_deterministic", dev, *args, ws.data_ptr())
        else:
            _lib.call("fiery_voxels_summing_forward", dev, *args)
        ctx.save_for_backward(seg)
        ctx.in_dtype = x.dtype
        ctx.channels = channels
        ctx.mark_non_differentiable(kept)
        return sums.to(x.dtype), kept.to(geometry.dtype)

    @staticmethod
    def backward(ctx, grad_x, grad_geometry):
        (seg,) = ctx.saved_tensors
        n_rows, channels = seg.shape[0], ctx.channels
        g = grad_x.float().contiguous()
        out = torch.empty((n_rows, channels), dtype=torch.float32, device=g.device)
        _lib.call("fiery_voxels_summing_backward", g.device, n_rows, channels, g.data_ptr(), seg.data_ptr(), out.data_ptr())
        return out.to(ctx.in_dtype), None, None
