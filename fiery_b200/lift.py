"""The fused camera->BEV lift behind the reference's call signatures.

Reference call sites replaced (SURVEY.md section 8b):
  (B3) ``Fiery.calculate_birds_eye_view_features(x, intrinsics, extrinsics) -> (b, s, C, X, Y)``
       fiery/models/fiery.py:275-286 -- everything after ``Encoder.depth_layer`` (encoder.py:96) runs in the CUDA
       library: get_geometry (fiery.py:193-208), the softmax x context outer product (encoder.py:98-102) and
       projection_to_birds_eye_view / VoxelsSumming (fiery.py:221-273, geometry.py:283-314).
  (B1) ``VoxelsSumming.apply`` -- see fiery_b200/geometry.py.

``LiftSplat`` carries what ``Fiery.__init__`` builds for this path (fiery.py:18-29): the frustum and the three BEV
grid tensors, under the same names, so a reference ``state_dict`` loads into it unchanged.

The plain lift (``LiftSplat.forward``) and the lift with the warp in its layout pass (``LiftSplat.forward_warped``) run through one
dispatcher operator, ``torch.ops.fiery_b200.lift_splat`` (fiery_b200/ops.py: autograd formula, fake implementation, autocast rule,
and the choice of a geometry plan for the backward).  This module holds the C-ABI launches behind it.
"""
from __future__ import annotations

import collections
import os
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import _require_cuda
from .geometry import _unfilled, bev_offset_fp32, calculate_birds_eye_view_parameters, create_frustum, split_frustum, z_valid_interval

# The geometry plan's byte layout (fiery_b200/csrc/lift_plan.cuh): one record per (frame, camera, 4-column tile), then the touched
# maps (one byte per frame and pillar).  A record holds mask[192] u32, off[192] u16, soff[64] u16, the counts (n_runs, n_stream) u32
# in 16 bytes, runs[192 * 32] i32 and streams[192 * 32 + 2 * 64] i32, padded to 128 bytes.
_PLAN_OFF_COUNTS = 192 * 4 + 192 * 2 + 64 * 2
_PLAN_TILE_BYTES = (_PLAN_OFF_COUNTS + 16 + 192 * 32 * 4 + (192 * 32 + 2 * 64) * 4 + 127) // 128 * 128


def _plan_touched_offset(n_frames: int, n_cameras: int, feat_w: int) -> int:
    """Byte offset of the touched maps in a plan of ``n_frames`` frames: the end of the tile records."""
    return n_frames * n_cameras * ((feat_w + 3) // 4) * _PLAN_TILE_BYTES


def _plan_bytes(n_frames, n_cameras, feat_w: int, pillars: int):
    """fiery_lift_plan_bytes: the tile records, then the touched maps rounded up to 128 bytes (0 for 0 frames).  Integer arithmetic
    only, so ``n_frames`` / ``n_cameras`` may be SymInts (the operator's fake implementation sizes the plan it returns with it)."""
    return _plan_touched_offset(n_frames, n_cameras, feat_w) + (n_frames * pillars + 127) // 128 * 128


_TORCH_TO_DTYPE = {torch.float32: _lib.DTYPE_F32, torch.float16: _lib.DTYPE_F16}

# Half-precision head tensors (AMP, baseline.yml PRECISION 16): False (default) = the tensor is widened to fp32 on the device
# first and takes the TMA path; True = the forward tile kernel reads the fp16 tensor itself (cp.async pieces widened in shared
# memory).  Both compute the same fp32 arithmetic on exactly converted values.  The 8-byte cp.async pieces slow the tile kernel
# down by more than the widening pass costs, so widening stays the default.
# Overridable with FIERY_B200_NATIVE_FP16=0/1.
NATIVE_FP16_FORWARD = os.environ.get("FIERY_B200_NATIVE_FP16", "0") == "1"


def pack_sequence_dim(x: torch.Tensor) -> torch.Tensor:
    """(b, s, ...) -> (b*s, ...); fiery/utils/network.py:5-7."""
    b, s = x.shape[:2]
    return x.view(b * s, *x.shape[2:])


def unpack_sequence_dim(x: torch.Tensor, b: int, s: int) -> torch.Tensor:
    """(b*s, ...) -> (b, s, ...); fiery/utils/network.py:10-11."""
    return x.view(b, s, *x.shape[1:])


class _ScratchPool:
    """Zero-initialised accumulation buffers, one per (device, stream, size).  The kernels leave a buffer all-zero
    again when they finish (include/fiery_b200.h), so it is allocated and cleared once.  At most ``max_entries`` buffers
    are kept (least recently used first out); a call that fails drops its buffer (``discard``), because a launch sequence that
    stopped half way may have left it dirty."""

    def __init__(self, max_entries: int = 4):
        self._bufs: "collections.OrderedDict[Tuple[int, int, int], torch.Tensor]" = collections.OrderedDict()
        self.max_entries = max_entries

    @staticmethod
    def _key(device: torch.device, nbytes: int):
        return (device.index if device.index is not None else torch.cuda.current_device(),
                torch.cuda.current_stream(device).cuda_stream, nbytes)

    def get(self, device: torch.device, nbytes: int) -> torch.Tensor:
        key = self._key(device, nbytes)
        buf = self._bufs.get(key)
        if buf is None:
            buf = torch.zeros(nbytes // 4, dtype=torch.float32, device=device)
            self._bufs[key] = buf
            while len(self._bufs) > self.max_entries:
                self._bufs.popitem(last=False)       # the evicted tensor is freed once its queued work has run (caching allocator)
        else:
            self._bufs.move_to_end(key)
        return buf

    def discard(self, device: torch.device, nbytes: int) -> None:
        self._bufs.pop(self._key(device, nbytes), None)

    def clear(self) -> None:
        self._bufs.clear()


_scratch = _ScratchPool()


class LiftSplat(nn.Module):
    """Frustum + BEV grid constants of the lift and its forward/backward entry points.

    Parameter names (``frustum``, ``bev_resolution``, ``bev_start_position``, ``bev_dimension``) and shapes are those
    of ``Fiery`` (fiery/models/fiery.py:21-23,128) so reference checkpoints keep loading.
    """

    def __init__(self, x_bound=(-50.0, 50.0, 0.5), y_bound=(-50.0, 50.0, 0.5), z_bound=(-10.0, 10.0, 20.0),
                 d_bound=(2.0, 50.0, 1.0), final_dim=(224, 480), encoder_downsample: int = 8, out_channels: int = 64,
                 use_depth_distribution: bool = True, output_layout: str = "contiguous", calibration: str = "fused"):
        super().__init__()
        res, start, dim = calculate_birds_eye_view_parameters(list(x_bound), list(y_bound), list(z_bound))
        self.bev_resolution = nn.Parameter(res, requires_grad=False)
        self.bev_start_position = nn.Parameter(start, requires_grad=False)
        self.bev_dimension = nn.Parameter(dim, requires_grad=False)
        self.frustum = nn.Parameter(create_frustum(tuple(final_dim), encoder_downsample, list(d_bound)), requires_grad=False)
        self.encoder_out_channels = out_channels
        self.use_depth_distribution = use_depth_distribution
        if output_layout not in ("contiguous", "channels_last"):
            raise ValueError("output_layout must be 'contiguous' (what the reference returns) or 'channels_last'")
        if calibration not in ("fused", "torch"):
            raise ValueError("calibration must be 'fused' (R @ K^-1 composed in the kernel) or 'torch'")
        self.output_layout = output_layout
        self.calibration = calibration
        self._consts = None     # cached device-side constants, rebuilt when parameters move / change

    @classmethod
    def from_config(cls, cfg, **kw) -> "LiftSplat":
        """``cfg``: a fiery_b200.synthetic.LiftConfig, or a reference CfgNode-like object with LIFT / IMAGE / MODEL."""
        if hasattr(cfg, "LIFT"):
            return cls(cfg.LIFT.X_BOUND, cfg.LIFT.Y_BOUND, cfg.LIFT.Z_BOUND, cfg.LIFT.D_BOUND, cfg.IMAGE.FINAL_DIM,
                       cfg.MODEL.ENCODER.DOWNSAMPLE, cfg.MODEL.ENCODER.OUT_CHANNELS,
                       cfg.MODEL.ENCODER.USE_DEPTH_DISTRIBUTION, **kw)
        return cls(cfg.x_bound, cfg.y_bound, cfg.z_bound, cfg.d_bound, cfg.final_dim, cfg.downsample, cfg.out_channels,
                   cfg.use_depth_distribution, **kw)

    @classmethod
    def from_fiery(cls, model, **kw) -> "LiftSplat":
        """Adopts the constants of an instantiated reference ``Fiery`` module.  The four Parameters are SHARED with the model
        (same tensors), so a checkpoint loaded into the model afterwards, ``model.to(...)`` or an in-place edit is seen here:
        the device-side constants are re-derived whenever the tensors' storage or version changes (``_param_key``)."""
        self = cls.__new__(cls)
        nn.Module.__init__(self)
        as_param = lambda t: t if isinstance(t, nn.Parameter) else nn.Parameter(t, requires_grad=False)   # noqa: E731
        self.bev_resolution = as_param(model.bev_resolution)
        self.bev_start_position = as_param(model.bev_start_position)
        self.bev_dimension = as_param(model.bev_dimension)
        self.frustum = as_param(model.frustum)
        self.encoder_out_channels = int(model.encoder_out_channels)
        enc = getattr(model, "encoder", None)
        self.use_depth_distribution = bool(getattr(enc, "use_depth_distribution", True))
        self.output_layout = kw.get("output_layout", "contiguous")
        self.calibration = kw.get("calibration", "fused")
        self._consts = None
        return self

    # -- constants ------------------------------------------------------------------------------------------------
    def _apply(self, fn, *a, **k):
        self._consts = None
        return super()._apply(fn, *a, **k)

    def _param_key(self):
        """Identity + in-place version of the four constant tensors: load_state_dict / .data edits / copy_ change it."""
        return tuple((p.data_ptr(), p._version, str(p.device), tuple(p.shape))
                     for p in (self.frustum, self.bev_resolution, self.bev_start_position, self.bev_dimension))

    @torch.compiler.disable      # host bookkeeping (parameters read back with numpy): runs eagerly, never compiled into a graph
    def _constants(self, device: torch.device):
        c = self._consts
        key = self._param_key()
        if c is not None and c["device"] == device and c["key"] == key:
            return c
        u, v, d = split_frustum(self.frustum)
        dim = [int(x) for x in self.bev_dimension.detach().cpu().tolist()]
        res = self.bev_resolution.detach().float().cpu().numpy().astype(np.float32)
        off = bev_offset_fp32(self.bev_start_position, self.bev_resolution)
        z_lo, z_hi = z_valid_interval(float(res[2]), dim[2])
        c = dict(device=device, key=key, u=u.to(device), v=v.to(device), d=d.to(device), dim=dim, res=res, off=off,
                 z_lo=float(z_lo), z_hi=float(z_hi), D=int(d.numel()), h=int(v.numel()), w=int(u.numel()))
        self._consts = c
        return c

    def _desc(self, c, n_frames: int, n_cameras: int, head_dtype: torch.dtype, calib_mode: int, layout: int) -> _lib.LiftDesc:
        if head_dtype not in _TORCH_TO_DTYPE:
            raise _lib.FieryError(f"head dtype {head_dtype} is not supported (float32 / float16)")
        d = _lib.LiftDesc()
        d.n_frames, d.n_cameras = n_frames, n_cameras
        d.depth_bins, d.channels = c["D"], self.encoder_out_channels
        d.feat_h, d.feat_w = c["h"], c["w"]
        d.bev_x, d.bev_y, d.bev_z = c["dim"]
        for a in range(3):
            d.bev_offset[a] = float(c["off"][a])
            d.bev_resolution[a] = float(c["res"][a])
        d.z_valid_lo, d.z_valid_hi = c["z_lo"], c["z_hi"]
        d.use_depth_distribution = 1 if self.use_depth_distribution else 0
        d.head_dtype = _TORCH_TO_DTYPE[head_dtype]
        d.calib_mode = calib_mode
        d.bev_layout = layout
        return d

    def _calibration(self, intrinsics: torch.Tensor, extrinsics: torch.Tensor):
        """Returns (calib_mode, a, b) device tensors for the C ABI."""
        if self.calibration == "torch":
            # the reference's own expression (fiery.py:196,203) on the inputs' device; inv_ex avoids the host sync of
            # torch.inverse's error check and runs the same LAPACK/cuSOLVER routine
            rotation, translation = extrinsics[..., :3, :3], extrinsics[..., :3, 3]
            combined = rotation.matmul(torch.linalg.inv_ex(intrinsics).inverse)
            return _lib.CALIB_COMPOSED, combined.float().contiguous(), translation.float().contiguous()
        return _lib.CALIB_RAW, intrinsics.float().contiguous(), extrinsics.float().contiguous()

    def _abi_args(self, dev: torch.device, intrinsics: torch.Tensor, extrinsics: torch.Tensor, head_dtype: torch.dtype, layout: int):
        """(descriptor, geometry) of a C-ABI call on these calibrations (B', n, ...) on ``dev``: ``geometry`` is the five tensors
        behind the calls' geometry pointers (calibration a and b, frustum u, v and d).  Hold it until the call is queued: the
        calibration pair may be a temporary."""
        c = self._constants(dev)
        mode, a, b = self._calibration(intrinsics.to(dev), extrinsics.to(dev))
        B, n = intrinsics.shape[:2]
        return self._desc(c, B, n, head_dtype, mode, layout), (a, b, c["u"], c["v"], c["d"])

    @staticmethod
    def _check_plan(plan: Optional[torch.Tensor], desc: _lib.LiftDesc, dev: torch.device) -> None:
        """A caller-owned plan must be the buffer ``plan()`` makes for this call's (B', n): exactly ``_plan_bytes`` bytes of uint8
        on ``dev`` (one byte for B' = 0).  The kernels find the touched maps at an offset computed from this call's frame count, so a
        plan of another batch would be read at the wrong place, not merely out of range."""
        if plan is None:
            return
        want = max(1, _plan_bytes(desc.n_frames, desc.n_cameras, desc.feat_w, desc.bev_x * desc.bev_y))
        if plan.dtype != torch.uint8 or plan.device != dev or plan.numel() != want:
            raise ValueError("plan was made for another batch shape: rebuild it with LiftSplat.plan(intrinsics, extrinsics)")

    # -- public entry points --------------------------------------------------------------------------------------
    def forward(self, head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor,
                plan: Optional[torch.Tensor] = None, warp: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> torch.Tensor:
        """head (B'*n, D+C, h, w) [= Encoder.depth_layer output, encoder.py:96], intrinsics (B', n, 3, 3),
        extrinsics (B', n, 4, 4) -> BEV features (B', C, X, Y) float32 (fiery.py:225-227 allocates float32).
        ``plan``: the geometry of this calibration from ``self.plan(intrinsics, extrinsics)`` -- pass it while the camera rig
        is static and the per-call geometry pass disappears; ``None`` computes it inside the call.
        ``warp``: (theta (B', 2, 3) float32, copy_mask (B',) uint8) samples every frame under its map in the layout pass (see
        ``forward_warped``); the BEV is then NCHW whatever ``output_layout`` says."""
        from . import ops
        _require_cuda(head, "head")                     # loud and specific: the operators are registered for CUDA only
        make_plan = plan is None and torch.is_grad_enabled() and head.requires_grad      # a training step shares one plan
        bev, _plan = torch.ops.fiery_b200.lift_splat(head, intrinsics, extrinsics, plan, ops.register_module(self, head.device), make_plan,
                                                     *(warp if warp is not None else (None, None)))
        return bev

    def forward_warped(self, head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor, flow: torch.Tensor,
                       spatial_extent, plan: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The lift followed by ``cumulative_warp_features(bev.clone(), flow, mode='bilinear', spatial_extent=...)``
        (fiery.py:140-146) as ONE chain: ``flow`` (b, s, 6) is the sequence's egomotion, ``intrinsics`` / ``extrinsics`` are
        (b*s, n, ...), ``head`` (b*s*n, D+C, h, w); returns (b, s, C, X, Y) float32 contiguous.  The layout pass gathers the
        bilinear neighbours of every output pixel straight from the channel-last accumulator (fiery_lift_forward_warped), so the
        unwarped BEV is never written.  Backward: the warp's adjoint, then the lift's backward (one shared plan)."""
        from .warp import _device_theta
        _require_cuda(head, "head")
        b, s = flow.shape[:2]
        if intrinsics.shape[0] != b * s:
            raise ValueError(f"flow is (b={b}, s={s}, 6) but the calibrations hold {intrinsics.shape[0]} frames")
        if s == 1:                                         # identity, like the reference (geometry.py:237)
            return self.forward(head, intrinsics, extrinsics, plan).unflatten(0, (b, s)).contiguous()
        if flow.shape[1] < 2:
            raise IndexError("flow needs at least two timesteps")
        warp = _device_theta(flow.to(head.device), spatial_extent, cumulative=True)
        return self.forward(head, intrinsics, extrinsics, plan, warp).unflatten(0, (b, s))

    def plan(self, intrinsics: torch.Tensor, extrinsics: torch.Tensor) -> torch.Tensor:
        """The geometry plan of a batch of calibrations (fiery_lift_plan): where every frustum point lands -- get_geometry
        (fiery.py:193-208) + voxel index / mask / rank (fiery.py:236-256) -- as pillar runs, in a device byte tensor.  Valid for
        forward and backward calls with the same (B', n) and these calibrations.  A call rejects a plan whose size is not that
        of its own (B', n) (``ValueError``); a plan of the same size made by another module, BEV grid or frustum, or for other
        calibrations, cannot be detected and gives a wrong BEV."""
        _require_cuda(intrinsics, "intrinsics")
        dev = intrinsics.device
        desc, geo = self._abi_args(dev, intrinsics, extrinsics, torch.float32, _lib.BEV_NCHW)
        buf = torch.empty(max(1, _plan_bytes(desc.n_frames, desc.n_cameras, desc.feat_w, desc.bev_x * desc.bev_y)), dtype=torch.uint8,
                          device=dev)
        _lib.call("fiery_lift_plan", dev, desc, *(t.data_ptr() for t in geo), buf.data_ptr())
        return buf

    def point_indices(self, intrinsics: torch.Tensor, extrinsics: torch.Tensor):
        """Integer voxel coordinates of every frustum point, as the reference computes them at fiery.py:236-256.
        Returns (idx (B', N, 3) int64, valid (B', N) bool, pillar (B', N) int32 [rank, or -1 if masked])."""
        _require_cuda(intrinsics, "intrinsics")
        dev = intrinsics.device
        desc, geo = self._abi_args(dev, intrinsics, extrinsics, torch.float32, _lib.BEV_NCHW)
        B, N = desc.n_frames, desc.n_cameras * desc.depth_bins * desc.feat_h * desc.feat_w
        idx = torch.empty((B, N, 3), dtype=torch.int64, device=dev)
        valid = torch.empty((B, N), dtype=torch.uint8, device=dev)
        pillar = torch.empty((B, N), dtype=torch.int32, device=dev)
        _lib.call("fiery_lift_point_indices", dev, desc, *(t.data_ptr() for t in geo), idx.data_ptr(), valid.data_ptr(),
                  pillar.data_ptr())
        return idx, valid.bool(), pillar

    def compose_calibration(self, intrinsics: torch.Tensor, extrinsics: torch.Tensor):
        """combined = R @ inverse(K) and translation (fiery.py:196,203) from the device kernel."""
        _require_cuda(intrinsics, "intrinsics")
        dev = intrinsics.device
        K = intrinsics.float().contiguous()
        E = extrinsics.float().contiguous()
        lead = K.shape[:-2]
        n = int(np.prod(lead)) if len(lead) else 1
        comb = torch.empty(lead + (3, 3), dtype=torch.float32, device=dev)
        trans = torch.empty(lead + (3,), dtype=torch.float32, device=dev)
        _lib.call("fiery_compose_calibration", dev, n, K.data_ptr(), E.data_ptr(), comb.data_ptr(), trans.data_ptr())
        return comb, trans

    def plan_summary(self, plan: torch.Tensor, n_frames: int, n_cameras: int) -> Dict[str, int]:
        """Counts read back from a plan buffer (layout: fiery_b200/csrc/lift_plan.cuh): pillar runs, backward stream entries and
        pillars that receive a point.  Diagnostic (bench.py uses it for the per-kernel algorithmic bytes); synchronises."""
        c = self._constants(plan.device)
        X, Y, _ = c["dim"]
        if plan.numel() != max(1, _plan_bytes(n_frames, n_cameras, c["w"], X * Y)):
            raise ValueError(f"plan holds {plan.numel()} bytes, not those of {n_frames} frames of {n_cameras} cameras")
        t0 = _plan_touched_offset(n_frames, n_cameras, c["w"])
        records = plan[:t0].view(t0 // _PLAN_TILE_BYTES, _PLAN_TILE_BYTES)
        counts = records[:, _PLAN_OFF_COUNTS:_PLAN_OFF_COUNTS + 8].contiguous().view(torch.int32)
        touched = plan[t0:t0 + n_frames * X * Y]
        return {"runs": int(counts[:, 0].sum()), "stream_entries": int(counts[:, 1].sum()), "touched_pillars": int(touched.ne(0).sum()),
                "tile_record_bytes": _PLAN_TILE_BYTES}

    # -- CUDA graph and host-buffer entry points ------------------------------------------------------------------------
    def capture(self, head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor,
                static_calibration: bool = False) -> "GraphedLift":
        """Captures one forward lift of these (device-resident, static) tensors into a CUDA graph.  ``g = lift.capture(...)``;
        ``bev = g()`` replays it: one graph launch instead of descriptor encoding + kernel launches from Python.
        ``static_calibration=True``: the calibration tensors never change between replays (a fixed camera rig), so the geometry
        plan is computed once here and the replay only runs the tile kernels and layout passes; otherwise the plan kernels are
        part of every replay.  The returned BEV tensor is the graph's static output buffer (overwritten by the next replay).
        Inference only."""
        return GraphedLift(self, head, intrinsics, extrinsics, static_calibration)

    def lift_from_host(self, head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor,
                       out: Optional[torch.Tensor] = None, device: Optional[torch.device] = None,
                       chunk_frames=3) -> torch.Tensor:
        """Host-buffer entry point: ``head`` (B'*n, D+C, h, w), ``intrinsics`` (B', n, 3, 3), ``extrinsics`` (B', n, 4, 4) in
        (pinned) host memory -> BEV (B', C, X, Y) in pinned host memory.  Frames are independent, so the batch is cut into
        chunks of ``chunk_frames`` and the three stages -- host->device copy, lift, device->host copy -- run on three
        streams, overlapping the upload of chunk i+1 and the download of chunk i-1 with the lift of chunk i (PCIe is
        full duplex).  ``chunk_frames`` may be a sequence: the sizes of the first chunks (the last entry repeats) -- a small first
        chunk starts the download earlier, and the download of 82 MB per 8 frames is what bounds the call.  Synchronises before
        returning.  Inference only."""
        dev = device if device is not None else next(self.parameters()).device
        if dev.type != "cuda":
            raise _lib.FieryError("lift_from_host needs the module on a CUDA device: fiery_b200 has no CPU path")
        c = self._constants(dev)
        B, n = intrinsics.shape[:2]
        C = self.encoder_out_channels
        X, Y, _ = c["dim"]
        if out is None:
            out = torch.empty((B, C, X, Y), dtype=torch.float32).pin_memory()
        st = self._host_streams(dev)
        cur = torch.cuda.current_stream(dev)
        for s in st:
            s.wait_stream(cur)
        up, run, down = st
        prev_done = None
        sizes = [max(1, int(c)) for c in (chunk_frames if isinstance(chunk_frames, (list, tuple)) else [chunk_frames])]
        bounds, f0 = [], 0
        while f0 < B:
            n_here = sizes[min(len(bounds), len(sizes) - 1)]
            bounds.append((f0, min(B, f0 + n_here)))
            f0 += n_here
        with torch.no_grad():
            for f0, f1 in bounds:
                with torch.cuda.stream(up):
                    h = head[f0 * n:f1 * n].to(dev, non_blocking=True)
                    k = intrinsics[f0:f1].to(dev, non_blocking=True)
                    e = extrinsics[f0:f1].to(dev, non_blocking=True)
                    ready = torch.cuda.Event()
                    ready.record(up)
                with torch.cuda.stream(run):
                    run.wait_event(ready)
                    bev = self._launch_forward(h, k, e)
                    for t in (h, k, e):
                        t.record_stream(run)
                    done = torch.cuda.Event()
                    done.record(run)
                with torch.cuda.stream(down):
                    down.wait_event(done)
                    out[f0:f1].copy_(bev, non_blocking=True)
                    bev.record_stream(down)
        cur.wait_stream(down)
        down.synchronize()
        return out

    def _host_streams(self, dev):
        key = (dev.index if dev.index is not None else torch.cuda.current_device())
        cache = self.__dict__.setdefault("_streams", {})
        if key not in cache:
            cache[key] = tuple(torch.cuda.Stream(device=dev) for _ in range(3))
        return cache[key]

    # -- raw launches (used by the operators in ops.py and by bench.py) ----------------------------------------------
    def _launch_forward(self, head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor,
                        scratch: Optional[torch.Tensor] = None, plan: Optional[torch.Tensor] = None,
                        warp: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> torch.Tensor:
        """``warp``: (theta (B', 2, 3), copy_mask (B',) uint8) -- the layout pass samples every frame under its map
        (fiery_lift_forward_warped); NCHW output only.
        Under ``torch.use_deterministic_algorithms(True)`` the call runs the bit-reproducible forward
        (fiery_lift_forward_deterministic: every pillar's runs added in a fixed order, no atomics) in a workspace of its own;
        ``scratch`` is then unused."""
        _require_cuda(head, "head")
        lib = _lib.load()
        dev = head.device
        c = self._constants(dev)
        if intrinsics.dim() != 4 or extrinsics.dim() != 4:
            raise ValueError("intrinsics must be (B', n, 3, 3) and extrinsics (B', n, 4, 4)")
        B, n = intrinsics.shape[:2]
        C = self.encoder_out_channels
        ch = C + (c["D"] if self.use_depth_distribution else 0)
        if tuple(head.shape) != (B * n, ch, c["h"], c["w"]):
            raise ValueError(f"head must be {(B * n, ch, c['h'], c['w'])}, got {tuple(head.shape)}")
        if head.dtype != torch.float32 and not (head.dtype == torch.float16 and NATIVE_FP16_FORWARD):
            head = head.float()                      # half-precision heads: widen first (see NATIVE_FP16_FORWARD)
        head = head.contiguous()
        nhwc = self.output_layout == "channels_last" and warp is None
        desc, geo = self._abi_args(dev, intrinsics, extrinsics, head.dtype, _lib.BEV_NHWC if nhwc else _lib.BEV_NCHW)
        self._check_plan(plan, desc, dev)
        X, Y, _ = c["dim"]
        if warp is not None:
            theta, copy_mask = warp
            if theta.numel() != B * 6 or copy_mask.numel() != B or theta.dtype != torch.float32 or copy_mask.dtype != torch.uint8:
                raise ValueError("warp must be (theta (B', 2, 3) float32, copy_mask (B',) uint8) for the B' frames of this call")
        warp_ptrs = (theta.data_ptr(), copy_mask.data_ptr()) if warp is not None else (0, 0)
        shape = (B, X, Y, C) if nhwc else (B, C, X, Y)
        pooled = 0
        if torch.are_deterministic_algorithms_enabled():
            entry, extra = "fiery_lift_forward_deterministic", warp_ptrs
            store = _unfilled(shape, torch.float32, dev)                      # every element is written
            buf = _unfilled(max(1, int(lib.fiery_lift_deterministic_workspace_bytes(desc))), torch.uint8, dev)
        else:
            entry, extra = ("fiery_lift_forward_warped", warp_ptrs) if warp is not None else ("fiery_lift_forward", ())
            # NHWC: the tile kernels reduce into the output itself, so it starts zeroed
            store = (torch.zeros if nhwc else torch.empty)(shape, dtype=torch.float32, device=dev)
            buf = scratch
            if buf is None and B and not nhwc:
                pooled = int(lib.fiery_lift_scratch_bytes(desc))
                buf = _scratch.get(dev, pooled)            # zero-filled once; the kernels leave it zeroed again
        try:
            _lib.call(entry, dev, desc, head.data_ptr(), *(t.data_ptr() for t in geo), store.data_ptr(),
                      buf.data_ptr() if (B and buf is not None) else 0, plan.data_ptr() if plan is not None else 0, *extra)
        except _lib.FieryError:
            if pooled:
                _scratch.discard(dev, pooled)          # a launch sequence that stopped half way may have left it dirty
            raise
        return store.permute(0, 3, 1, 2) if nhwc else store

    def _launch_backward(self, head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor,
                         grad_bev: torch.Tensor, plan: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Gradient of the BEV w.r.t. ``head``, in ``head``'s dtype; the backward kernel reads the head widened to fp32."""
        dev = head.device
        h32 = head.float().contiguous()
        g = grad_bev.float()
        if g.permute(0, 2, 3, 1).is_contiguous() and not g.is_contiguous():
            layout = _lib.BEV_NHWC
        else:
            layout = _lib.BEV_NCHW
            g = g.contiguous()
        desc, geo = self._abi_args(dev, intrinsics, extrinsics, torch.float32, layout)
        self._check_plan(plan, desc, dev)
        grad_head = torch.empty_like(h32)
        ws = None
        if plan is None or layout == _lib.BEV_NCHW:        # re-layout of an NCHW gradient and/or room for the plan records
            ws = torch.empty(max(1, int(_lib.load().fiery_lift_workspace_bytes(desc)) // 4), dtype=torch.float32, device=dev)
        _lib.call("fiery_lift_backward", dev, desc, h32.data_ptr(), *(t.data_ptr() for t in geo), g.data_ptr(), grad_head.data_ptr(),
                  ws.data_ptr() if ws is not None else 0, plan.data_ptr() if plan is not None else 0)
        return grad_head.to(head.dtype)


class GraphedLift:
    """A captured forward lift (see ``LiftSplat.capture``)."""

    def __init__(self, module: LiftSplat, head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor,
                 static_calibration: bool = False):
        _require_cuda(head, "head")
        self.module, self.inputs = module, (head, intrinsics, extrinsics)
        dev = head.device
        self.plan = module.plan(intrinsics, extrinsics) if static_calibration and intrinsics.shape[0] else None
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(2):                       # warm-up outside capture: attribute setup, scratch allocation
                module._launch_forward(head, intrinsics, extrinsics, plan=self.plan)
        torch.cuda.current_stream(dev).wait_stream(side)
        # the graph owns its accumulation scratch (zeroed once here; every replay leaves it zeroed again)
        self.scratch = None
        if module.output_layout != "channels_last" and intrinsics.shape[0]:
            desc, _ = module._abi_args(dev, intrinsics, extrinsics, head.dtype, _lib.BEV_NCHW)
            self.scratch = torch.zeros(int(_lib.load().fiery_lift_scratch_bytes(desc)) // 4, dtype=torch.float32, device=dev)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph), torch.no_grad():
            self.output = module._launch_forward(head, intrinsics, extrinsics, scratch=self.scratch, plan=self.plan)

    def __call__(self) -> torch.Tensor:
        self.graph.replay()
        return self.output


def _head_and_lift(self, x, intrinsics, extrinsics):
    """The part of fiery.py:275-286 in front of the lift: backbone + depth_layer on the packed cameras, and this model's LiftSplat."""
    b, s, n, c, h, w = x.shape
    x = pack_sequence_dim(x)
    intrinsics = pack_sequence_dim(intrinsics)
    extrinsics = pack_sequence_dim(extrinsics)
    enc = self.encoder
    head = enc.depth_layer(enc.get_features(x.view(b * s * n, c, h, w)))          # encoder.py:94-96
    lift = getattr(self, "_fiery_b200_lift", None)
    if lift is None:
        lift = LiftSplat.from_fiery(self)          # shares the model's Parameters; device-side constants follow them
        object.__setattr__(self, "_fiery_b200_lift", lift)
    return head, intrinsics, extrinsics, lift


def calculate_birds_eye_view_features(self, x, intrinsics, extrinsics):
    """Replacement for ``Fiery.calculate_birds_eye_view_features`` (fiery/models/fiery.py:275-286), same signature:
    x (b, s, n, 3, H, W), intrinsics (b, s, n, 3, 3), extrinsics (b, s, n, 4, 4) -> (b, s, C, X, Y).

    ``self`` is the reference ``Fiery`` module; its backbone and ``depth_layer`` (library convolutions,
    encoder.py:94-96) run unchanged, everything after them runs in the fused CUDA lift."""
    b, s = x.shape[:2]
    head, intrinsics, extrinsics, lift = _head_and_lift(self, x, intrinsics, extrinsics)
    bev = lift(head, intrinsics, extrinsics)
    return unpack_sequence_dim(bev, b, s)


def birds_eye_view_features_warped(self, x, intrinsics, extrinsics, future_egomotion):
    """``Fiery.forward``'s two statements fiery.py:140-146 in one call:

        x = self.calculate_birds_eye_view_features(image, intrinsics, extrinsics)
        x = cumulative_warp_features(x.clone(), future_egomotion, mode='bilinear', spatial_extent=self.spatial_extent)

    -> (b, s, C, X, Y): the past frames' BEV features in the present frame's reference, the present frame as is.  The warp runs
    as the lift's layout pass (``LiftSplat.forward_warped``), so the unwarped BEV is never materialised; INTEGRATION.md shows the
    two-line patch of ``Fiery.forward``."""
    head, intrinsics, extrinsics, lift = _head_and_lift(self, x, intrinsics, extrinsics)
    return lift.forward_warped(head, intrinsics, extrinsics, future_egomotion, tuple(float(v) for v in self.spatial_extent))
