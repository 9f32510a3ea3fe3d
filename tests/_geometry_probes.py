"""Frustum points placed on the decision boundaries of the point -> pillar map (fiery/models/fiery.py:236-247), for the tests of
every path that evaluates it (tests/test_geometry_envelope_gpu.py) and their CPU check (tests/test_geometry_probes_cpu.py).

A case is a BEV grid, the separable frustum factors u (columns), v (rows), d (depths) and a composed calibration (combined,
translation) per (frame, camera), chosen so that the ego position of every point is set by the test:
  * boundary cases: camera 0 is the identity, so at depth 1 the point (u, v, 1) carries an x probe on its column and a y probe on
    its row; camera 1 keeps x and y inside the grid and puts the depth factor on z, so the depths carry the z probes.
  * run-pattern cases: the row coordinate v takes a few values (inside cell A, inside cell B, out of range, NaN); four cameras
    map them to y so that the same rows read as pillar changes and returns, valid -> masked and masked -> valid, and no change.
Probe values are found by searching the ordered fp32 values through the oracle's explicit fp32 chain (oracle.lift_oracle:
frustum_to_ego_explicit, voxel_indices_explicit) for the first float past each boundary, as fiery_b200.geometry.z_valid_interval
finds the z interval; the neighbours are nextafter steps from there."""
from __future__ import annotations

import dataclasses
from typing import List, Tuple

import numpy as np
import torch

from fiery_b200.geometry import bev_offset_fp32, z_valid_interval
from oracle import lift_oracle as O

f32 = np.float32
C = 64                      # the only channel count the lift accepts
INT64_EDGE = 2.0 ** 63


@dataclasses.dataclass
class Grid:
    name: str
    x_bound: Tuple[float, float, float]
    y_bound: Tuple[float, float, float]
    z_bound: Tuple[float, float, float] = (-10.0, 10.0, 20.0)

    def __post_init__(self):
        res, start, dim = O.bev_grid(self.x_bound, self.y_bound, self.z_bound)      # fiery/utils/geometry.py:53-56
        self.res = res.numpy().astype(f32)
        self.start = start.numpy().astype(f32)
        self.dim = dim.numpy().astype(np.int64)
        self.off = bev_offset_fp32(start, res)                                        # fiery.py:236
        self.z_lo, self.z_hi = z_valid_interval(float(self.res[2]), int(self.dim[2]))
        self.X, self.Y = int(self.dim[0]), int(self.dim[1])

    def interior(self, a: int) -> f32:
        """An ego coordinate well inside the grid on axis a (z: inside the valid height interval)."""
        if a == 2:
            return f32(self.off[2] + f32(0.5) * self.res[2])
        k = self.dim[a] // 3
        return f32(self.off[a] + (k + 0.5) * self.res[a])

    def scaled(self, ego: np.ndarray) -> np.ndarray:
        """s = (p - offset) / res in fp32 (fiery.py:236), the value .long() truncates."""
        with np.errstate(invalid="ignore", over="ignore"):
            return ((ego.astype(f32) - self.off).astype(f32) / self.res).astype(f32)

    def indices(self, ego: np.ndarray):
        """The oracle's explicit chain: (idx (..., 3) int64, keep (...)) of ego points (..., 3)."""
        with np.errstate(invalid="ignore", over="ignore"):
            return O.voxel_indices_explicit(ego, self.start, self.res, self.dim)


GRIDS = {
    # both horizontal resolutions powers of two: the scale is an exact multiply (PillarMap<true>); x starts at 0, so s reaches
    # every float just above -1
    "pow2": Grid("pow2", (0.0, 16.0, 0.5), (-4.0, 4.0, 0.25)),
    # neither: true division (PillarMap<false>)
    "div": Grid("div", (-15.0, 15.0, 0.3), (-10.5, 10.5, 0.7)),
    # x a power of two, y not: the division instantiation, with one axis exact
    "mixed": Grid("mixed", (0.0, 16.0, 0.5), (-9.0, 9.0, 0.3)),
    # X*Y odd: the NCHW layout pass that is not TMA
    "odd": Grid("odd", (-7.0, 7.0, 0.4), (-10.5, 10.5, 1.0)),
}
GRID_DIMS = {"pow2": (32, 32), "div": (100, 30), "mixed": (32, 60), "odd": (35, 21)}

# X (or Y) above 2^24, where float(X) rounds to the nearest float: 2^24 + 1 rounds down to 2^24 (the case that was wrong),
# 2^24 is exact and 2^24 + 3 rounds up
EDGE = 2 ** 24
BIG_GRIDS = {
    "x2p24p1": Grid("x2p24p1", (0.0, float(EDGE + 1), 1.0), (0.0, 1.0, 1.0)),
    "y2p24p1": Grid("y2p24p1", (0.0, 1.0, 1.0), (0.0, float(EDGE + 1), 1.0)),
    "x2p24": Grid("x2p24", (0.0, float(EDGE), 1.0), (0.0, 1.0, 1.0)),
    "x2p24p3": Grid("x2p24p3", (0.0, float(EDGE + 3), 1.0), (0.0, 1.0, 1.0)),
}
BIG_DIMS = {"x2p24p1": (EDGE + 1, 1), "y2p24p1": (1, EDGE + 1), "x2p24": (EDGE, 1), "x2p24p3": (EDGE + 3, 1)}


# ---- probes on one axis --------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Probe:
    """An ego coordinate p on one axis.  keep / idx: what the explicit chain gives (idx None: unspecified, s not finite or
    |s| >= 2^63).  step (+1 / -1 / 0): the nextafter neighbour in that direction crosses the boundary the probe sits on, to
    n_keep / n_idx.  exact: the probe's s (x, y) or p - offset (z) equals this value exactly."""
    label: str
    p: f32
    keep: bool
    idx: object
    step: int = 0
    n_keep: bool = False
    n_idx: object = None
    exact: object = None


def _nudge(p, direction):
    return np.nextafter(f32(p), f32(np.inf) if direction > 0 else f32(-np.inf), dtype=f32)


def _axis_eval(grid: Grid, a: int, p) -> Tuple[int, bool, f32]:
    ego = np.array([grid.interior(0), grid.interior(1), grid.interior(2)], dtype=f32)
    ego[a] = f32(p)
    idx, keep = grid.indices(ego[None])
    return int(idx[0, a]), bool(keep[0]), grid.scaled(ego[None])[0, a]


def _key(p) -> int:
    """Position of a float32 in the ordered sequence of float32 values (+-0 share 0): consecutive floats, consecutive keys."""
    i = int(np.array(f32(p)).view(np.int32))
    return i if i >= 0 else -(i & 0x7FFFFFFF)


def _val(k: int) -> f32:
    bits = k if k >= 0 else (-k) | 0x80000000
    return np.array(bits & 0xFFFFFFFF, dtype=np.uint32).view(f32)[()]


def _first(pred, guess) -> f32:
    """Smallest float p with pred(p) (pred monotone: false below, true above): a bracket around guess, then bisection over the
    ordered floats (walking one ulp at a time would cross the 2^24 subnormals next to zero)."""
    k = _key(guess)
    step = 1
    if pred(_val(k)):
        hi, lo = k, k - 1
        while pred(_val(lo)):
            hi, step = lo, step * 2
            lo = k - step
    else:
        lo, hi = k, k + 1
        while not pred(_val(hi)):
            lo, step = hi, step * 2
            hi = k + step
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if pred(_val(mid)):
            hi = mid
        else:
            lo = mid
    return _val(hi)


def _spec(s) -> bool:
    return bool(np.isfinite(s)) and abs(float(s)) < INT64_EDGE


def axis_probes(grid: Grid, a: int) -> List[Probe]:
    """Probes on horizontal axis a (0 = x, 1 = y): the mask edges s = -1, the band -1 < s < 0, s = N and one ulp below, cell
    edges, NaN, +-inf and huge values."""
    N = int(grid.dim[a])
    off, res = float(grid.off[a]), float(grid.res[a])
    ev = lambda p: _axis_eval(grid, a, p)                                   # noqa: E731
    kept = lambda p: ev(p)[1]                                               # noqa: E731
    out: List[Probe] = []

    def add(label, p, step=0, exact=None):
        i, k, s = ev(p)
        n_i, n_k = (None, False)
        if step:
            n_i, n_k, _ = ev(_nudge(p, step))
        out.append(Probe(label, f32(p), k, i if _spec(s) else None, step, n_k, n_i, exact))

    p0 = _first(lambda p: ev(p)[2] > -1.0, off - res)                        # first point kept at the low edge: trunc(s) = 0
    add("first_kept", p0, step=-1)
    pm1 = _first(lambda p: ev(p)[2] >= -1.0, off - res)
    if ev(pm1)[2] == -1.0:
        add("s_eq_-1", pm1, step=+1, exact=-1.0)
    add("band_mid", f32(off - 0.5 * res))                                    # -1 < s < 0 truncates to cell 0
    pz = _first(lambda p: ev(p)[2] >= 0.0, off)
    add("band_top", _nudge(pz, -1))                                        # largest s < 0: still cell 0
    add("s_ge_0", pz)
    for k in sorted({1, N // 2, N - 1}):
        if 1 <= k <= N - 1:
            pk = _first(lambda p: ev(p)[0] >= k, off + k * res)
            add(f"edge_{k}", pk, step=-1)
            add(f"below_edge_{k}", _nudge(pk, -1), step=+1)
    pN = _first(lambda p: ev(p)[0] >= N and ev(p)[2] >= N, off + N * res)   # first point past the top: s >= N
    add("last_kept", _nudge(pN, -1), step=+1)
    add("s_ge_N", pN, step=-1, exact=float(N) if ev(pN)[2] == N else None)
    add("interior", grid.interior(a))
    for label, p in (("nan", np.nan), ("+inf", np.inf), ("-inf", -np.inf), ("+max", np.finfo(f32).max),
                     ("-max", -np.finfo(f32).max), ("s_1e10", off + 1e10 * res), ("s_-1e10", off - 1e10 * res),
                     ("s_1e20", off + 1e20 * res), ("s_-1e20", off - 1e20 * res)):
        add(label, f32(p))
    assert all(kept(q.p) == q.keep for q in out)
    return out


def z_probes(grid: Grid) -> List[Probe]:
    """Probes on z: the ends of the valid interval [z_lo, z_hi] of p - offset_z, one ulp either side, and non-finite values."""
    ev = lambda p: _axis_eval(grid, 2, p)                                   # noqa: E731
    az = lambda p: f32(f32(p) - grid.off[2])                                # noqa: E731
    out: List[Probe] = []

    def add(label, p, step=0, exact=None):
        i, k, s = ev(p)
        n_i, n_k = (None, False)
        if step:
            n_i, n_k, _ = ev(_nudge(p, step))
        out.append(Probe(label, f32(p), k, i if _spec(s) else None, step, n_k, n_i, exact))

    lo = _first(lambda p: ev(p)[0] >= 0 and ev(p)[2] > -1.0, grid.off[2] + grid.z_lo)
    hi = _nudge(_first(lambda p: ev(p)[0] >= 1 or ev(p)[2] >= 1.0, grid.off[2] + grid.z_hi), -1)
    add("z_lo", lo, step=-1, exact=float(grid.z_lo) if az(lo) == grid.z_lo else None)
    add("z_lo_below", _nudge(lo, -1), step=+1)
    add("z_lo_above", _nudge(lo, +1))
    add("z_hi", hi, step=+1, exact=float(grid.z_hi) if az(hi) == grid.z_hi else None)
    add("z_hi_above", _nudge(hi, +1), step=-1)
    add("z_hi_below", _nudge(hi, -1))
    for label, p in (("nan", np.nan), ("+inf", np.inf), ("-inf", -np.inf), ("+max", np.finfo(f32).max)):
        add(label, f32(p))
    return out


# ---- cases ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    name: str
    grid: Grid
    u: np.ndarray                # (w,) column factors, w % 4 == 0
    v: np.ndarray                # (h,) row factors
    d: np.ndarray                # (D,) depth factors
    comb: np.ndarray             # (n, 3, 3) combined = R @ K^-1 of every camera (the same in every frame)
    trans: np.ndarray            # (n, 3)
    frame_shift: float = 0.0     # frame f adds f * frame_shift to every camera's x translation

    @property
    def n(self):
        return self.comb.shape[0]

    def calibration(self, frames: int):
        comb = np.broadcast_to(self.comb, (frames,) + self.comb.shape).astype(f32).copy()
        trans = np.broadcast_to(self.trans, (frames,) + self.trans.shape).astype(f32).copy()
        trans[..., 0] = (trans[..., 0] + (np.arange(frames, dtype=f32) * f32(self.frame_shift))[:, None]).astype(f32)
        return comb, trans

    def ego(self, frames: int) -> np.ndarray:
        """(frames, n, D, h, w, 3) ego positions by the explicit chain (fiery.py:199-205)."""
        comb, trans = self.calibration(frames)
        with np.errstate(invalid="ignore", over="ignore"):
            return O.frustum_to_ego_explicit(self.u, self.v, self.d, comb, trans)

    def oracle(self, frames: int):
        """idx (frames, n, D, h, w, 3) int64, keep (same without the 3) bool, pillar int32 (rank or -1), s (fp32 scaled coords)."""
        ego = self.ego(frames)
        idx, keep = self.grid.indices(ego)
        s = self.grid.scaled(ego)
        s[..., 2] = ((ego[..., 2] - self.grid.off[2]).astype(f32) / self.grid.res[2]).astype(f32)
        pillar = np.where(keep, idx[..., 0] * self.grid.Y + idx[..., 1], -1).astype(np.int64)
        assert int(pillar.max(initial=-1)) < self.grid.X * self.grid.Y
        return idx, keep, pillar.astype(np.int32), s


def _pad4(x: List[f32], fill) -> np.ndarray:
    x = list(x)
    while len(x) % 4:
        x.append(fill)
    return np.array(x, dtype=f32)


def boundary_case(grid: Grid) -> Case:
    xp, yp, zp = axis_probes(grid, 0), axis_probes(grid, 1), z_probes(grid)
    assert len(yp) <= 32
    u = _pad4([q.p for q in xp], grid.interior(0))
    v = np.array([q.p for q in yp], dtype=f32)
    d = np.array([1.0] + [q.p for q in zp] + [1.0], dtype=f32)
    comb = np.zeros((2, 3, 3), dtype=f32)
    trans = np.zeros((2, 3), dtype=f32)
    comb[0] = np.eye(3, dtype=f32)                               # camera 0: p = (u d, v d, d); at d = 1 exactly (u, v, 1)
    comb[0, 2, 2] = 0.0
    trans[0, 2] = grid.interior(2)                               # ... with z inside the valid interval
    comb[1, 2, 2] = 1.0                                          # camera 1: p = (x_in, y_in, d)
    trans[1, :2] = grid.interior(0), grid.interior(1)
    return Case(f"boundary-{grid.name}", grid, u, v, d, comb, trans)


# run patterns: y = v d + t_y per camera on a grid of 1 m cells with Y = 8
RUN_GRID = Grid("runs", (-16.0, 16.0, 0.5), (0.0, 8.0, 1.0))
RUN_A, RUN_B, RUN_OUT = 0.5, 2.5, 100.0
RUN_HS = (1, 2, 3, 4, 7, 8, 9, 16, 31, 32)
_MIXED = ("A", "A", "nan", "A", "out", "B", "A", "B", "B", "nan", "nan", "B", "out", "out", "A", "A")


def run_case(h: int, pattern: str) -> Case:
    """pattern 'alt': rows A, B, A, B, ...; 'mixed': a fixed draw from {A, B, out of range, NaN}.  Cameras (y = v d + t_y, d in
    [1, 1.75]): 0 keeps A and B in cells 0 and 2-4 (change, return), 1 moves B past Y (valid <-> masked), 2 moves A below 0
    (masked <-> valid), 3 ignores v (no change).  x = u d + t_x puts every (column, depth) pair in its own pillar."""
    code = {"A": RUN_A, "B": RUN_B, "out": RUN_OUT, "nan": np.nan}
    rows = ["A" if r % 2 == 0 else "B" for r in range(h)] if pattern == "alt" else [_MIXED[r % len(_MIXED)] for r in range(h)]
    v = np.array([code[r] for r in rows], dtype=f32)
    u = np.arange(8, dtype=f32) * f32(0.75)
    d = np.array([1.0, 1.25, 1.5, 1.75, 1.125], dtype=f32)
    comb = np.zeros((4, 3, 3), dtype=f32)
    trans = np.zeros((4, 3), dtype=f32)
    for cam, ty in enumerate((0.0, 6.0, -2.0, 3.5)):
        comb[cam, 0, 0] = 1.0
        comb[cam, 1, 1] = 0.0 if cam == 3 else 1.0
        trans[cam] = (-14.0, ty, RUN_GRID.interior(2))
    return Case(f"runs-h{h}-{pattern}", RUN_GRID, u, v, d, comb, trans, frame_shift=0.25)


def boundary_events(pillar: np.ndarray):
    """pillar (..., h, w) -> dict event -> (h,) bool: whether row boundary b (rows b-1 | b) hosts the event anywhere."""
    h = pillar.shape[-2]
    P = np.moveaxis(pillar, -2, 0).reshape(h, -1)
    ev = {k: np.zeros(h, dtype=bool) for k in ("change", "return", "valid_to_masked", "masked_to_valid", "no_change", "gap")}
    for b in range(1, h):
        a, c = P[b - 1], P[b]
        ev["change"][b] = bool(((a >= 0) & (c >= 0) & (a != c)).any())
        earlier = (P[:b - 1] == c[None]).any(0) if b >= 2 else np.zeros_like(c, dtype=bool)
        ev["return"][b] = bool(((c >= 0) & (a != c) & earlier).any())
        ev["valid_to_masked"][b] = bool(((a >= 0) & (c < 0)).any())
        ev["masked_to_valid"][b] = bool(((a < 0) & (c >= 0)).any())
        ev["no_change"][b] = bool(((a >= 0) & (a == c)).any())
        ev["gap"][b] = bool(((c >= 0) & (a < 0) & (P[b - 2] == c)).any()) if b >= 2 else False
    return ev


# ---- calibrations for the LU with partial pivoting of compose_camera ---------------------------------------------------------
def pivot_sequence(K: np.ndarray) -> Tuple[int, int]:
    """Pivot rows (step 0, step 1) the explicit LU (oracle.lift_oracle.compose_calibration_explicit) picks: first maximum."""
    a = np.asarray(K, dtype=f32).copy()
    piv = []
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for j in range(2):
            p = j + int(np.argmax(np.abs(a[j:, j])))
            piv.append(p)
            if p != j:
                a[[j, p]] = a[[p, j]]
            rcp = f32(1.0) / a[j, j]
            for i in range(j + 1, 3):
                a[i, j] = f32(a[i, j] * rcp)
            for i in range(j + 1, 3):
                for k in range(j + 1, 3):
                    a[i, k] = f32(a[i, k] - f32(a[i, j] * a[j, k]))
    return piv[0], piv[1]


def pivot_intrinsics():
    """(name, K, claim) with claim = the pivot sequence (p0, p1) for the finite cases, or 'singular' / 'nonfinite'."""
    out = []
    rng = np.random.default_rng(2024)
    want = {(p0, p1) for p0 in range(3) for p1 in range(1, 3)}
    while want:                                                  # small integers, every pivot order with a clear winner
        K = rng.integers(-9, 10, (3, 3)).astype(f32)
        if abs(float(np.linalg.det(K.astype(np.float64)))) < 1.0:
            continue
        seq = pivot_sequence(K)
        col0 = np.abs(K[:, 0])
        if seq in want and (np.sort(col0)[-1] > np.sort(col0)[-2]):
            want.discard(seq)
            out.append((f"pivots-{seq[0]}{seq[1]}", K, seq))
    ties = {
        # equal magnitudes of opposite sign: the first maximum wins
        "tie0-pos-first": np.array([[2, 1, 0], [-2, 3, 1], [1, 0, 4]], dtype=f32),
        "tie0-neg-first": np.array([[-3, 1, 2], [1, 2, 0], [3, 0, 1]], dtype=f32),
        "tie1": np.array([[4, 1, 2], [2, 3, 1], [2, -1, 5]], dtype=f32),
        "pinhole": np.array([[500.5, 0, 320.25], [0, 480.75, 240.5], [0, 0, 1]], dtype=f32),
        "pinhole-0.3": np.array([[0.3 * 1266.417, 0, 0.3 * 816.267], [0, 0.3 * 1266.417, 0.3 * 491.507 - 46], [0, 0, 1]], dtype=f32),
    }
    for name, K in ties.items():
        out.append((name, K, pivot_sequence(K)))
    singular = {
        "zero-col0": np.array([[0, 1, 2], [0, 3, 1], [0, 1, 4]], dtype=f32),       # zero pivot at step 0
        "rank2-step1": np.array([[1, 2, 3], [2, 4, 6], [1, 2, 4]], dtype=f32),     # zero pivot at step 1
        "rank2-step2": np.array([[1, 2, 3], [4, 5, 6], [7, 8, 9]], dtype=f32),     # pivot 0 at step 2
        "zeros": np.zeros((3, 3), dtype=f32),
    }
    for name, K in singular.items():
        out.append((name, K, "singular"))
    nonfinite = {
        "nan": np.array([[500, 0, 320], [0, np.nan, 240], [0, 0, 1]], dtype=f32),
        "inf": np.array([[np.inf, 0, 320], [0, 500, 240], [0, 0, 1]], dtype=f32),
        "inf-offdiag": np.array([[500, np.inf, 320], [0, 500, 240], [0, 0, 1]], dtype=f32),
    }
    for name, K in nonfinite.items():
        out.append((name, K, "nonfinite"))
    return out


def pivot_extrinsics(n: int, seed: int = 7) -> np.ndarray:
    """(n, 4, 4): a rotation about z by a dyadic-free angle and a translation (camera -> ego)."""
    rng = np.random.default_rng(seed)
    E = np.zeros((n, 4, 4), dtype=f32)
    for i in range(n):
        t = rng.uniform(-np.pi, np.pi)
        E[i, :3, :3] = [[np.cos(t), 0, np.sin(t)], [np.sin(t), 0, -np.cos(t)], [0, 1, 0]]
        E[i, :3, 3] = rng.uniform(-2, 2, 3)
        E[i, 3, 3] = 1
    return E


def torch_chain(case: Case, frames: int):
    """The reference chain on torch-CPU with the given combined: frustum_to_ego then voxel_indices, per frame."""
    comb, trans = case.calibration(frames)
    frustum = torch.stack(torch.broadcast_tensors(torch.from_numpy(case.u).view(1, 1, -1), torch.from_numpy(case.v).view(1, -1, 1),
                                                  torch.from_numpy(case.d).view(-1, 1, 1)), -1).contiguous()
    E = torch.zeros(frames, case.n, 4, 4)
    E[..., :3, 3] = torch.from_numpy(trans)
    E[..., :3, :3] = torch.eye(3)
    E[..., 3, 3] = 1
    K = torch.eye(3).expand(frames, case.n, 3, 3).contiguous()
    ego = O.frustum_to_ego(frustum, K, E, combined=torch.from_numpy(comb))
    g = case.grid
    res, start, dim = torch.from_numpy(g.res), torch.from_numpy(g.start), torch.from_numpy(g.dim)
    out = [O.voxel_indices(ego[f], start, res, dim) for f in range(frames)]
    return ego.numpy(), torch.stack([o[0] for o in out]).numpy(), torch.stack([o[1] for o in out]).numpy()
