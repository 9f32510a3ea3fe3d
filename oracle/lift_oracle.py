"""CPU oracle for the camera->BEV lift.  TEST INFRASTRUCTURE ONLY.

This file is a CPU restatement (torch-CPU / numpy) of the reference's Lift-Splat hot path.  It exists so that
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline leg can check / time the algorithm on a
machine without the reference.  Nothing under ``fiery_b200/`` may import it: the product path
is the CUDA library and fails loudly without it.

Where the arithmetic lives: the reference (wayveai/fiery @ fd03f16) is pure Python calling PyTorch
(pinned ``pytorch=1.7.0`` in ``environment.yml:8``; this container runs torch 2.11).  Results are defined by
these torch calls: ``softmax`` (encoder.py:99), ``inverse``/``matmul`` (fiery.py:203-204), ``.long()``
truncation (fiery.py:237), ``argsort`` (fiery.py:257), ``cumsum`` (geometry.py:289), ``index_put``
(fiery.py:265).  The oracle calls the same torch-CPU primitives in the same order, so it *is* the reference's
algorithm on this torch build; ``oracle/gen_golden.py`` checks it against the real reference bytecode imported
from a reference checkout (``FIERY_REFERENCE``) and commits golden vectors under ``tests/golden/``.

Pinned: the reference ships no tests or fixtures (SURVEY.md section 4), so parity is pinned by (i) golden
vectors generated from the reference's own functions by ``oracle/gen_golden.py`` and (ii) the live
oracle-vs-reference comparison that script performs.  See tests/test_oracle_golden.py.

Every function cites the reference lines it follows.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
import torch


# --------------------------------------------------------------------------------------------------------
# a7: BEV grid constants                                  fiery/utils/geometry.py:39-58
# --------------------------------------------------------------------------------------------------------
def bev_grid(x_bound: Sequence[float], y_bound: Sequence[float], z_bound: Sequence[float]):
    """(resolution f32[3], first-cell-centre f32[3], dimension i64[3]).  geometry.py:53-56: python-float
    arithmetic, then ``torch.tensor`` (f32) / truncating cast to long."""
    rows = (x_bound, y_bound, z_bound)
    resolution = torch.tensor([r[2] for r in rows])
    start = torch.tensor([r[0] + r[2] / 2.0 for r in rows])
    dimension = torch.tensor([(r[1] - r[0]) / r[2] for r in rows], dtype=torch.long)
    return resolution, start, dimension


# --------------------------------------------------------------------------------------------------------
# a1: frustum                                              fiery/models/fiery.py:109-128
# --------------------------------------------------------------------------------------------------------
def frustum_grid(final_dim: Tuple[int, int], downsample: int, d_bound: Sequence[float]) -> torch.Tensor:
    """(D, h, w, 3) tensor of (u_pixel, v_pixel, depth); fiery.py:115-127."""
    H, W = final_dim
    fh, fw = H // downsample, W // downsample
    depth = torch.arange(*d_bound, dtype=torch.float)                       # fiery.py:115
    D = depth.shape[0]
    u = torch.linspace(0, W - 1, fw, dtype=torch.float)                     # fiery.py:120
    v = torch.linspace(0, H - 1, fh, dtype=torch.float)                     # fiery.py:122
    grid = torch.empty(D, fh, fw, 3, dtype=torch.float)
    grid[..., 0] = u.view(1, 1, fw)
    grid[..., 1] = v.view(1, fh, 1)
    grid[..., 2] = depth.view(D, 1, 1)
    return grid


# --------------------------------------------------------------------------------------------------------
# a2: frustum -> ego frame                                 fiery/models/fiery.py:193-208
# --------------------------------------------------------------------------------------------------------
def compose_calibration(intrinsics: torch.Tensor, extrinsics: torch.Tensor):
    """``combined = R @ inverse(K)`` (fiery.py:203) and ``translation`` (fiery.py:196), shapes (B,n,3,3),(B,n,3)."""
    rotation = extrinsics[..., :3, :3]
    translation = extrinsics[..., :3, 3]
    return rotation.matmul(torch.inverse(intrinsics)), translation


def compose_calibration_explicit(intrinsics: np.ndarray, extrinsics: np.ndarray):
    """numpy restatement of fiery.py:196,203 with every fp32 operation written out -- the arithmetic of
    ``compose_camera`` in fiery_b200/csrc/geometry.cuh.  ``inverse`` follows the published LAPACK route torch's CPU
    ``linalg.inv`` takes (solve against the identity): sgetf2 (partial pivoting, first maximum, column scaled by the
    reciprocal pivot) then sgetrs/strsm (forward substitution with the unit-lower factor, back substitution with
    true division by the diagonal); ``R @ Kinv`` accumulates k = 0,1,2 without FMA.  Bit-equal to torch-CPU for
    pinhole (upper-triangular) intrinsics -- checked in tests/test_oracle_golden.py; a few ulp off for general 3x3.

    intrinsics (...,3,3), extrinsics (...,4,4) -> combined (...,3,3), translation (...,3), float32."""
    f32 = np.float32
    Ks = np.asarray(intrinsics, dtype=f32).reshape(-1, 3, 3)
    Es = np.asarray(extrinsics, dtype=f32).reshape(-1, 4, 4)
    comb = np.empty((Ks.shape[0], 3, 3), dtype=f32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for m in range(Ks.shape[0]):
            a = Ks[m].copy()
            b = np.eye(3, dtype=f32)
            for j in range(3):
                p = j + int(np.argmax(np.abs(a[j:, j])))
                if p != j:
                    a[[j, p]] = a[[p, j]]
                    b[[j, p]] = b[[p, j]]
                rcp = f32(1.0) / a[j, j]
                for i in range(j + 1, 3):
                    a[i, j] = f32(a[i, j] * rcp)
                for i in range(j + 1, 3):
                    for k in range(j + 1, 3):
                        a[i, k] = f32(a[i, k] - f32(a[i, j] * a[j, k]))
            for c in range(3):
                for k in range(3):
                    for i in range(k + 1, 3):
                        b[i, c] = f32(b[i, c] - f32(a[i, k] * b[k, c]))
                for k in range(2, -1, -1):
                    b[k, c] = f32(b[k, c] / a[k, k])
                    for i in range(k):
                        b[i, c] = f32(b[i, c] - f32(a[i, k] * b[k, c]))
            R = Es[m, :3, :3]
            for i in range(3):
                for j in range(3):
                    acc = f32(R[i, 0] * b[0, j])
                    acc = f32(acc + f32(R[i, 1] * b[1, j]))
                    acc = f32(acc + f32(R[i, 2] * b[2, j]))
                    comb[m, i, j] = acc
    lead = np.asarray(intrinsics).shape[:-2]
    return comb.reshape(lead + (3, 3)), Es[:, :3, 3].copy().reshape(lead + (3,))


def frustum_to_ego(frustum: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor,
                   combined: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(B, n, D, h, w, 3) ego-frame xyz of every frustum point; fiery.py:199-205.

    ``combined`` may be supplied to pin ``R @ K^-1`` to a particular LAPACK/cuSOLVER result (SURVEY.md section 7,
    hard part 2-iv)."""
    comb, trans = compose_calibration(intrinsics, extrinsics)
    if combined is not None:
        comb = combined
    B, n = trans.shape[:2]
    pts = frustum.view(1, 1, *frustum.shape, 1)                             # (1,1,D,h,w,3,1)   fiery.py:199
    pix_times_depth = pts[..., :2, :] * pts[..., 2:3, :]                    # (u*d, v*d)        fiery.py:202
    homog = torch.cat((pix_times_depth, pts[..., 2:3, :]), dim=5)
    ego = comb.view(B, n, 1, 1, 1, 3, 3).matmul(homog).squeeze(-1)          # fiery.py:204
    ego = ego + trans.view(B, n, 1, 1, 1, 3)                                # fiery.py:205 (in-place there)
    return ego


def frustum_to_ego_explicit(u: np.ndarray, v: np.ndarray, depth: np.ndarray, combined: np.ndarray,
                            translation: np.ndarray) -> np.ndarray:
    """numpy restatement with the floating-point order written out; this is the arithmetic the CUDA kernels
    implement and SURVEY.md appendix A found bit-equal to torch-CPU's batched 3x3 @ 3x1:

        p_r = (((M[r,0]*(u*d)) + (M[r,1]*(v*d))) + (M[r,2]*d)) + t_r          individually rounded f32, no FMA

    u (w,), v (h,), depth (D,), combined (B,n,3,3), translation (B,n,3) -> (B,n,D,h,w,3) float32."""
    f32 = np.float32
    u, v, depth = u.astype(f32), v.astype(f32), depth.astype(f32)
    ud = (u[None, None, :] * depth[:, None, None]).astype(f32)              # (D,1,w)
    vd = (v[None, :, None] * depth[:, None, None]).astype(f32)              # (D,h,1)
    dd = depth[:, None, None]
    M = combined.astype(f32)[:, :, None, None, None]                        # (B,n,1,1,1,3,3)
    t = translation.astype(f32)[:, :, None, None, None]
    out = np.empty(combined.shape[:2] + (depth.size, v.size, u.size, 3), dtype=f32)
    for r in range(3):
        acc = (M[..., r, 0] * ud).astype(f32)
        acc = (acc + (M[..., r, 1] * vd).astype(f32)).astype(f32)
        acc = (acc + (M[..., r, 2] * dd).astype(f32)).astype(f32)
        out[..., r] = (acc + t[..., r]).astype(f32)
    return out


# --------------------------------------------------------------------------------------------------------
# a3 + a4: depth distribution x context                    fiery/models/encoder.py:98-102, fiery.py:216-217
# --------------------------------------------------------------------------------------------------------
def depth_context_volume(head: torch.Tensor, n_cameras: int, D: int, C: int,
                         use_depth_distribution: bool = True) -> torch.Tensor:
    """head (B*n, D+C, h, w) -> (B, n, D, h, w, C) view of the outer product (encoder.py:99-100) or of the
    uniform-depth repeat (encoder.py:102)."""
    if use_depth_distribution:
        prob = head[:, :D].softmax(dim=1)                                   # encoder.py:99
        vol = prob.unsqueeze(1) * head[:, D:D + C].unsqueeze(2)             # encoder.py:100  (B*n,C,D,h,w)
    else:
        vol = head.unsqueeze(2).repeat(1, 1, D, 1, 1)                       # encoder.py:102
    vol = vol.view(vol.shape[0] // n_cameras, n_cameras, *vol.shape[1:])    # fiery.py:216
    return vol.permute(0, 1, 3, 4, 5, 2)                                    # fiery.py:217


# --------------------------------------------------------------------------------------------------------
# a5 (first half): voxel indices                            fiery/models/fiery.py:236-247
# --------------------------------------------------------------------------------------------------------
def voxel_indices(ego_b: torch.Tensor, start: torch.Tensor, resolution: torch.Tensor, dimension: torch.Tensor):
    """One frame: ego_b (n,D,h,w,3) -> (idx (N,3) int64 [truncation toward zero], keep (N,) bool)."""
    scaled = (ego_b - (start - resolution / 2.0)) / resolution               # fiery.py:236
    idx = scaled.view(-1, 3).long()                                          # fiery.py:237
    keep = ((idx[:, 0] >= 0) & (idx[:, 0] < dimension[0])                    # fiery.py:240-247
            & (idx[:, 1] >= 0) & (idx[:, 1] < dimension[1])
            & (idx[:, 2] >= 0) & (idx[:, 2] < dimension[2]))
    return idx, keep


def voxel_indices_explicit(ego: np.ndarray, start: np.ndarray, resolution: np.ndarray, dimension: np.ndarray):
    """numpy restatement of fiery.py:236-247 with the f32 order written out: sub, true division, trunc."""
    f32 = np.float32
    offset = (start.astype(f32) - (resolution.astype(f32) / f32(2.0)).astype(f32)).astype(f32)
    scaled = ((ego.astype(f32) - offset).astype(f32) / resolution.astype(f32)).astype(f32)
    with np.errstate(invalid="ignore"):
        idx = np.trunc(scaled).astype(np.int64)
    keep = np.ones(idx.shape[:-1], dtype=bool)
    for a in range(3):
        keep &= (idx[..., a] >= 0) & (idx[..., a] < int(dimension[a]))
    return idx, keep


# --------------------------------------------------------------------------------------------------------
# a6: VoxelsSumming                                         fiery/utils/geometry.py:283-314
# --------------------------------------------------------------------------------------------------------
class CumsumSegmentSum(torch.autograd.Function):
    """Segmented sum over rank-sorted rows by global prefix sum and adjacent difference."""

    @staticmethod
    def forward(ctx, feats, coords, ranks):
        prefix = feats.cumsum(0)                                             # geometry.py:289
        last_of_run = torch.ones(prefix.shape[0], device=prefix.device, dtype=torch.bool)
        last_of_run[:-1] = ranks[1:] != ranks[:-1]                           # geometry.py:292-293
        prefix, coords = prefix[last_of_run], coords[last_of_run]            # geometry.py:295
        sums = torch.cat((prefix[:1], prefix[1:] - prefix[:-1]))             # geometry.py:297
        ctx.save_for_backward(last_of_run)
        ctx.mark_non_differentiable(coords)                                  # geometry.py:300
        return sums, coords

    @staticmethod
    def backward(ctx, grad_sums, grad_coords):
        (last_of_run,) = ctx.saved_tensors
        seg = torch.cumsum(last_of_run, 0)                                   # geometry.py:309
        seg[last_of_run] -= 1                                                # geometry.py:310
        return grad_sums[seg], None, None                                    # geometry.py:312-314


def direct_segment_sum(feats: torch.Tensor, ranks: torch.Tensor, dtype=torch.float64):
    """Numerical ground truth for a6: per-segment sums accumulated directly in ``dtype`` (no prefix sums)."""
    if feats.shape[0] == 0:
        return feats.new_zeros((0, feats.shape[1]), dtype=dtype)
    boundary = torch.ones(feats.shape[0], dtype=torch.bool)
    boundary[1:] = ranks[1:] != ranks[:-1]
    seg = torch.cumsum(boundary, 0) - 1
    out = torch.zeros(int(seg[-1]) + 1, feats.shape[1], dtype=dtype)
    out.index_add_(0, seg, feats.to(dtype))
    return out


# --------------------------------------------------------------------------------------------------------
# a5 (second half): splat                                   fiery/models/fiery.py:221-273
# --------------------------------------------------------------------------------------------------------
def splat(vol: torch.Tensor, ego: torch.Tensor, start, resolution, dimension) -> torch.Tensor:
    """vol (B,n,D,h,w,C), ego (B,n,D,h,w,3) -> BEV (B,C,X,Y) float32.  Per-frame loop as in fiery.py:231."""
    B = vol.shape[0]
    C = vol.shape[-1]
    X, Y, Z = (int(d) for d in dimension)
    bev = torch.zeros((B, C, X, Y), dtype=torch.float, device=vol.device)   # fiery.py:225-227
    n_pts = vol[0].numel() // C
    for b in range(B):
        feats = vol[b].reshape(n_pts, C)                                     # fiery.py:233
        idx, keep = voxel_indices(ego[b], start, resolution, dimension)
        feats, idx = feats[keep], idx[keep]                                  # fiery.py:248-249
        ranks = idx[:, 0] * (Y * Z) + idx[:, 1] * Z + idx[:, 2]              # fiery.py:252-256
        order = ranks.argsort()                                              # fiery.py:257
        feats, idx, ranks = feats[order], idx[order], ranks[order]           # fiery.py:258
        feats, idx = CumsumSegmentSum.apply(feats, idx, ranks)               # fiery.py:261
        cells = torch.zeros((Z, X, Y, C), device=feats.device)              # fiery.py:263
        cells[idx[:, 2], idx[:, 0], idx[:, 1]] = feats                       # fiery.py:265
        bev[b] = cells.permute((0, 3, 1, 2)).squeeze(0)                      # fiery.py:268-271 (needs Z == 1)
    return bev


# --------------------------------------------------------------------------------------------------------
# a8: the whole region {head, intrinsics, extrinsics} -> BEV      fiery/models/fiery.py:275-286
# --------------------------------------------------------------------------------------------------------
class LiftOracle:
    """Holds the constants ``Fiery.__init__`` builds (fiery.py:18-29) and runs the lift on CPU."""

    def __init__(self, final_dim=(224, 480), downsample=8, out_channels=64, x_bound=(-50.0, 50.0, 0.5),
                 y_bound=(-50.0, 50.0, 0.5), z_bound=(-10.0, 10.0, 20.0), d_bound=(2.0, 50.0, 1.0),
                 use_depth_distribution=True):
        self.resolution, self.start, self.dimension = bev_grid(x_bound, y_bound, z_bound)
        self.frustum = frustum_grid(final_dim, downsample, d_bound)
        self.D = self.frustum.shape[0]
        self.C = out_channels
        self.use_depth_distribution = use_depth_distribution

    def to(self, device) -> "LiftOracle":
        """Moves the constants so the same torch op chain runs on another device (oracle variant O2 of SURVEY.md section 8c:
        the reference's ops executed on the GPU by torch's own library kernels -- a baseline, never the product)."""
        self.resolution, self.start = self.resolution.to(device), self.start.to(device)
        self.dimension, self.frustum = self.dimension.to(device), self.frustum.to(device)
        return self

    @classmethod
    def from_config(cls, cfg) -> "LiftOracle":
        return cls(cfg.final_dim, cfg.downsample, cfg.out_channels, cfg.x_bound, cfg.y_bound, cfg.z_bound,
                   cfg.d_bound, cfg.use_depth_distribution)

    def geometry(self, intrinsics, extrinsics, combined=None):
        return frustum_to_ego(self.frustum, intrinsics, extrinsics, combined)

    def lift(self, head: torch.Tensor, intrinsics: torch.Tensor, extrinsics: torch.Tensor,
             combined: Optional[torch.Tensor] = None) -> torch.Tensor:
        """head (B*n, D+C, h, w), intrinsics (B,n,3,3), extrinsics (B,n,4,4) -> (B, C, X, Y)."""
        n = intrinsics.shape[1]
        ego = self.geometry(intrinsics, extrinsics, combined)
        vol = depth_context_volume(head, n, self.D, self.C, self.use_depth_distribution)
        return splat(vol, ego, self.start, self.resolution, self.dimension)

    def point_indices(self, intrinsics, extrinsics, combined=None):
        """Per-frame integer voxel coordinates of all N points and their validity: (B,N,3) int64, (B,N) bool."""
        ego = self.geometry(intrinsics, extrinsics, combined)
        out = [voxel_indices(ego[b], self.start, self.resolution, self.dimension) for b in range(ego.shape[0])]
        return torch.stack([o[0] for o in out]), torch.stack([o[1] for o in out])

    def lift_exact(self, head, intrinsics, extrinsics, combined=None, dtype=torch.float64) -> torch.Tensor:
        """Ground truth (oracle variant O3 of SURVEY.md section 8c): same indices, but softmax, outer product and
        pooling done in float64 with a direct scatter-add -- adjudicates the reference's cumsum rounding."""
        n = intrinsics.shape[1]
        idx, keep = self.point_indices(intrinsics, extrinsics, combined)
        vol = depth_context_volume(head.to(dtype), n, self.D, self.C, self.use_depth_distribution)
        B = vol.shape[0]
        X, Y, _ = (int(d) for d in self.dimension)
        bev = torch.zeros(B, X * Y, self.C, dtype=dtype)
        for b in range(B):
            feats = vol[b].reshape(-1, self.C)[keep[b]]
            cell = idx[b][keep[b]]
            bev[b].index_add_(0, cell[:, 0] * Y + cell[:, 1], feats)
        return bev.view(B, X, Y, self.C).permute(0, 3, 1, 2).contiguous()


def normwise_error(a: torch.Tensor, truth: torch.Tensor) -> float:
    a, truth = a.detach().double(), truth.detach().double()
    return float((a - truth).norm() / truth.norm().clamp_min(1e-300))


def max_abs_scaled_error(a: torch.Tensor, truth: torch.Tensor) -> float:
    a, truth = a.detach().double(), truth.detach().double()
    return float((a - truth).abs().max() / truth.abs().max().clamp_min(1e-300))
