"""BEV feature warping behind the reference's signatures (SURVEY.md section 8f, next-1).

Mirrors, same names / arguments / return values:
  * ``warp_features(x, flow, mode='nearest', spatial_extent=None)``              fiery/utils/geometry.py:181-222
  * ``cumulative_warp_features(x, flow, mode='nearest', spatial_extent=None)``   fiery/utils/geometry.py:225-253
    (call site fiery/models/fiery.py:143-146 with ``mode='bilinear'``)

Two launches per call through the C ABI (fiery_b200/csrc/warp.cu): ``warp_theta_kernel`` evaluates the 6-DoF pose algebra
(``pose_vec2mat`` :145-160, ``euler2mat`` :110-142, the running product, ``mat2pose_vec`` :82-107; one thread per sequence, a
few 4x4 matrices) and ``warp_forward_kernel`` does the sampling -- ``affine_grid`` + ``grid_sample`` over the (b, C, X, Y)
feature maps, 10 MB per frame each way -- for all past frames of a sequence straight into the output tensor; the present
frame is copied.  No CPU path.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import _require_cuda


def _mode_flag(mode: str) -> int:
    if mode == "bilinear":
        return 0
    if mode == "nearest":
        return 1
    raise ValueError(f"mode must be 'bilinear' or 'nearest', got {mode!r}")


def _dense_maps(t: torch.Tensor) -> torch.Tensor:
    """(n, C, H, W) float32 with dense channel planes (any map stride)."""
    n, C, H, W = t.shape
    if t.dtype == torch.float32 and t.stride(3) == 1 and t.stride(2) == W and t.stride(1) == H * W:
        return t
    return t.float().contiguous()


class _WarpMaps(torch.autograd.Function):
    """x (n, C, H, W) sampled under theta (n, 2, 3); maps flagged in ``copy_mask`` (n,) uint8 pass through unchanged."""

    @staticmethod
    def forward(ctx, x, theta, copy_mask, nearest: int):
        _require_cuda(x, "x")
        n, C, H, W = x.shape
        xs = _dense_maps(x)
        th = theta.detach().float().contiguous()
        out = torch.empty((n, C, H, W), dtype=torch.float32, device=x.device)
        _lib.call("fiery_warp_features_forward", x.device, n, C, H, W, xs.data_ptr(), xs.stride(0) if n else 0, th.data_ptr(),
                  copy_mask.data_ptr() if copy_mask is not None else 0, out.data_ptr(), C * H * W, nearest)
        ctx.save_for_backward(th, copy_mask)
        ctx.nearest, ctx.dtype = nearest, x.dtype
        return out

    @staticmethod
    def backward(ctx, grad_out):
        th, mask = ctx.saved_tensors
        return _warp_adjoint(grad_out, th, mask, ctx.nearest).to(ctx.dtype), None, None, None


def _warp_adjoint(grad_out: torch.Tensor, theta: torch.Tensor, copy_mask, nearest: int) -> torch.Tensor:
    """Gradient (n, C, H, W) float32 of the maps sampled under theta (n, 2, 3) float32 w.r.t. their sources, for the upstream
    gradient ``grad_out`` (n, C, H, W); maps flagged in ``copy_mask`` (n,) uint8 or None pass it through (the gather adjoint,
    fiery_warp_features_backward).  Used by ``_WarpMaps`` and by the warped lift's backward (fiery_b200/ops.py)."""
    n, C, H, W = grad_out.shape
    g = _dense_maps(grad_out)
    grad_x = torch.empty((n, C, H, W), dtype=torch.float32, device=g.device)       # overwritten by the gather adjoint
    _lib.call("fiery_warp_features_backward", g.device, n, C, H, W, g.data_ptr(), g.stride(0) if n else 0, theta.data_ptr(),
              copy_mask.data_ptr() if copy_mask is not None else 0, grad_x.data_ptr(), C * H * W, nearest)
    return grad_x


def _device_theta(flow: torch.Tensor, spatial_extent, cumulative: bool):
    """theta (n, 2, 3) and copy mask (n,) for ``flow`` (b, 6) or, cumulative, (b, T, 6): fiery_warp_theta."""
    _require_cuda(flow, "flow")
    f = flow.detach().float().contiguous()
    b = f.shape[0]
    T = f.shape[1] if cumulative else 1
    theta = torch.empty((b * T, 2, 3), dtype=torch.float32, device=f.device)
    mask = torch.empty((b * T,), dtype=torch.uint8, device=f.device) if cumulative else None
    _lib.call("fiery_warp_theta", f.device, b, T, 1 if cumulative else 0, f.data_ptr(), float(spatial_extent[0]),
              float(spatial_extent[1]), theta.data_ptr(), mask.data_ptr() if cumulative else 0)
    return theta, mask


def warp_features(x: torch.Tensor, flow, mode: str = "nearest", spatial_extent=None) -> torch.Tensor:
    """Applies a z-rotation and xy translation to the feature map ``x (b, c, h, w)``; ``flow (b, 6)``; geometry.py:181-222.
    Like the sampling kernels, theta is computed without autograd (the reference never trains through egomotion)."""
    if flow is None:
        return x
    _require_cuda(x, "x")
    theta, _ = _device_theta(flow, spatial_extent, cumulative=False)
    res = _WarpMaps.apply(x, theta, None, _mode_flag(mode))
    return res if x.dtype == torch.float32 else res.to(x.dtype)


def cumulative_warp_features(x: torch.Tensor, flow: torch.Tensor, mode: str = "nearest", spatial_extent=None) -> torch.Tensor:
    """Warps a sequence ``x (b, t, c, h, w)`` by accumulating incremental egomotion ``flow (b, t, 6)``: x[:, -1] stays, x[:, t]
    is warped with flow[:, t] @ ... @ flow[:, -2]; geometry.py:225-253.  Two kernel launches produce the whole result (pose
    algebra; past frames sampled + present frame copied); the reference clones x, warps frame by frame and stacks."""
    b, T = x.shape[:2]
    if T == 1:
        return x
    _require_cuda(x, "x")
    F_len = flow.shape[1]
    if F_len < max(2, T - 1):
        raise IndexError(f"flow has {F_len} timesteps, the sequence {T}: the reference indexes flow[:, -2] and flow[:, t - 1]")
    if F_len != T:
        # the reference starts the running product at flow[:, -2] of flow's OWN length and continues with flow[:, t - 1]
        # indexed by the sequence's t (geometry.py:246-251): an effective per-frame sequence with that hybrid indexing
        flow = torch.cat([flow[:, :T - 2], flow[:, F_len - 2:F_len - 1], flow[:, F_len - 1:F_len]], dim=1)
    theta, copy_mask = _device_theta(flow, spatial_extent, cumulative=True)
    xm = x.reshape(b * T, *x.shape[2:])
    res = _WarpMaps.apply(xm, theta, copy_mask, _mode_flag(mode)).view(x.shape)
    return res if x.dtype == torch.float32 else res.to(x.dtype)
