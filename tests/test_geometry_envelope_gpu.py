"""GPU: the point -> pillar geometry (fiery/models/fiery.py:193-208,236-256) at its decision boundaries, on every path that
evaluates it, bit for bit against the oracle's explicit fp32 chain.

Four evaluators compute where a frustum point lands: pillar_of in point_indices_kernel, PillarMap + select_pillar in the plan
kernel, PillarMap inside the forward tile kernel's geometry stage (calls without a plan), and compose_camera for raw intrinsics.
Random calibrations almost never put a point on a decision boundary, so the cases here place them there on purpose
(tests/_geometry_probes.py, checked on the CPU by tests/test_geometry_probes_cpu.py): s = -1, the band -1 < s < 0, s = N and one ulp
below, cell edges under exact multiplication and true division, z_lo / z_hi and one ulp either side, NaN, +-inf and huge values;
and rows whose pillars change, return, leave and re-enter the grid or stay put at every row boundary, h from 1 to 32.

Every case runs through fiery_lift_point_indices, the decoded plan (ranks, touched map, backward streams), the forward without and
with a plan (both unit shapes of the tile kernel, NCHW and NHWC, fp32 and native fp16 heads), the warped forward and the backward
(NCHW and NHWC gradients, without and with a plan).  Heads hold small integers and depth logits of 0 for one bin and -200 for the
others (the softmax gives exact 1 / 0), or uniform depth, so every sum is exact and the outputs must EQUAL fp64 pooling at the
oracle's indices: a single misplaced point shows.  After every forward the scratch must be all zero again.

idx_out of fiery_lift_point_indices is unspecified where s is NaN, +-inf or |s| >= 2^63 (torch's .long() itself differs between
CPU and CUDA there); only valid = 0 and pillar = -1 are checked at those points."""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fiery_b200 import _lib
from oracle import lift_oracle as O
from tests import _geometry_probes as G
from tests._plan_layout import _decode, assert_tile_streams
from tests.test_lift_envelope_gpu import _unit_kernels

pytestmark = pytest.mark.gpu
C = G.C


def _dev():
    return torch.device("cuda:0")


def _stream():
    return torch.cuda.current_stream(_dev()).cuda_stream


def _ptr(t):
    return t.data_ptr() if t is not None else 0


# ---- cases ---------------------------------------------------------------------------------------------------------------------
BOUNDARY = {f"boundary-{n}": G.boundary_case(g) for n, g in G.GRIDS.items()}
RUNS = {f"runs-h{h}-{p}": G.run_case(h, p) for h in G.RUN_HS for p in ("alt", "mixed")}
CASES = {**BOUNDARY, **RUNS}


class Shape:
    """What tests/_plan_layout._decode reads from a config."""

    def __init__(self, case, frames):
        self.feat_hw = (case.v.size, case.u.size)
        self.depth_bins, self.n_cameras, self.frames = case.d.size, case.n, frames
        self.bev_hw = (case.grid.X, case.grid.Y)


def _desc(case, frames, use_depth=True, head_dtype=_lib.DTYPE_F32, layout=_lib.BEV_NCHW, calib=_lib.CALIB_COMPOSED):
    g = case.grid
    d = _lib.LiftDesc()
    d.n_frames, d.n_cameras, d.depth_bins, d.channels = frames, case.n, case.d.size, C
    d.feat_h, d.feat_w = case.v.size, case.u.size
    d.bev_x, d.bev_y, d.bev_z = g.X, g.Y, 1
    for a in range(3):
        d.bev_offset[a] = float(g.off[a])
        d.bev_resolution[a] = float(g.res[a])
    d.z_valid_lo, d.z_valid_hi = float(g.z_lo), float(g.z_hi)
    d.use_depth_distribution = 1 if use_depth else 0
    d.head_dtype, d.calib_mode, d.bev_layout = head_dtype, calib, layout
    return d


class Run:
    """Device inputs of one case at a frame count, and the oracle's answer."""

    def __init__(self, case, frames):
        self.case, self.frames = case, frames
        dev = _dev()
        comb, trans = case.calibration(frames)
        self.a = torch.from_numpy(comb).to(dev)
        self.b = torch.from_numpy(trans).to(dev)
        self.u, self.v, self.d = (torch.from_numpy(x).to(dev) for x in (case.u, case.v, case.d))
        self.idx, self.keep, self.pillar, self.s = case.oracle(frames)
        self.XY = case.grid.X * case.grid.Y
        self._heads = {}

    def frustum(self):
        return self.u.data_ptr(), self.v.data_ptr(), self.d.data_ptr()

    # heads: small-integer contexts; one-hot depth (logit 0 in one bin, -200 elsewhere) or uniform depth
    def head(self, mode):
        if mode not in self._heads:
            case, n_img = self.case, self.frames * self.case.n
            D, h, w = case.d.size, case.v.size, case.u.size
            rng = np.random.default_rng(zlib.crc32(f"{case.name}/{self.frames}/{mode}".encode()))
            ctx = rng.integers(1, 5, (n_img, C, h, w)) * rng.choice([-1, 1], (n_img, C, h, w))
            if mode == "onehot":
                hot = rng.integers(0, D, (n_img, h, w))
                logits = np.full((n_img, D, h, w), -200.0)
                np.put_along_axis(logits, hot[:, None], 0.0, axis=1)
                weight = (np.arange(D)[None, :, None, None] == hot[:, None]).astype(np.float64)
                head = np.concatenate([logits, ctx], 1)
            else:
                weight = np.ones((n_img, D, h, w))
                head = ctx
            self._heads[mode] = (torch.from_numpy(head.astype(np.float32)), torch.from_numpy(ctx.astype(np.float64)),
                                 torch.from_numpy(weight))
        return self._heads[mode]

    def pooled(self, mode):
        """fp64 pooling at the oracle's indices: (keys = frame * X*Y + pillar, sums (K, C)) of the pillars that receive points."""
        _, ctx, weight = self.head(mode)
        Fr, n, D, h, w = self.pillar.shape
        pil = torch.from_numpy(self.pillar.astype(np.int64))
        valid = pil >= 0
        key = pil + (torch.arange(Fr) * self.XY).view(Fr, 1, 1, 1, 1)
        vals = weight.view(Fr, n, D, h, w, 1) * ctx.view(Fr, n, C, h, w).permute(0, 1, 3, 4, 2).unsqueeze(2)
        keys, inv = torch.unique(key[valid], return_inverse=True)
        sums = torch.zeros(keys.numel(), C, dtype=torch.float64)
        sums.index_add_(0, inv, vals[valid])
        return keys, sums

    def expected_bev(self, mode):
        keys, sums = self.pooled(mode)
        out = torch.zeros(self.frames * self.XY, C, dtype=torch.float64)
        out[keys] = sums
        return out.view(self.frames, self.case.grid.X, self.case.grid.Y, C).permute(0, 3, 1, 2)

    def expected_grad(self, mode, gbev):
        """d<lift(head), gbev>/d head with exact 1 / 0 depth probabilities: context gradient = sum over depths of the weight times
        gbev at the point's pillar; logit gradient 0 (p (g_d - sum_k p_k g_k) vanishes for one-hot p)."""
        _, ctx, weight = self.head(mode)
        Fr, n, D, h, w = self.pillar.shape
        pil = torch.from_numpy(self.pillar.astype(np.int64))
        valid = pil >= 0
        key = torch.where(valid, pil + (torch.arange(Fr) * self.XY).view(Fr, 1, 1, 1, 1), torch.zeros_like(pil))
        gflat = gbev.double().permute(0, 2, 3, 1).reshape(-1, C)
        gathered = gflat[key] * (weight.view(Fr, n, D, h, w) * valid).unsqueeze(-1)
        gctx = gathered.sum(2).permute(0, 1, 4, 2, 3).reshape(Fr * n, C, h, w)
        if mode == "onehot":
            return torch.cat([torch.zeros(Fr * n, D, h, w, dtype=torch.float64), gctx], 1)
        return gctx

    # C ABI calls
    def point_indices(self):
        N = self.case.n * self.case.d.size * self.case.v.size * self.case.u.size
        dev = _dev()
        idx = torch.empty((self.frames, N, 3), dtype=torch.int64, device=dev)
        valid = torch.empty((self.frames, N), dtype=torch.uint8, device=dev)
        pillar = torch.empty((self.frames, N), dtype=torch.int32, device=dev)
        _lib.check(_lib.load().fiery_lift_point_indices(_desc(self.case, self.frames), _ptr(self.a), _ptr(self.b), *self.frustum(),
                                                        _ptr(idx), _ptr(valid), _ptr(pillar), _stream()), "fiery_lift_point_indices")
        shape = self.pillar.shape
        return idx.cpu().numpy().reshape(shape + (3,)), valid.cpu().numpy().reshape(shape), pillar.cpu().numpy().reshape(shape)

    def plan(self):
        lib = _lib.load()
        desc = _desc(self.case, self.frames)
        buf = torch.empty(int(lib.fiery_lift_plan_bytes(desc)), dtype=torch.uint8, device=_dev())
        _lib.check(lib.fiery_lift_plan(desc, _ptr(self.a), _ptr(self.b), *self.frustum(), _ptr(buf), _stream()), "fiery_lift_plan")
        return buf

    def forward(self, mode, half=False, layout=_lib.BEV_NCHW, plan=None, warp=None, out=None):
        """BEV (frames, C, X, Y) on the device in the logical layout; the NCHW scratch is checked to be all zero again."""
        lib = _lib.load()
        head = self.head(mode)[0].to(_dev())
        if half:
            head = head.half()
        desc = _desc(self.case, self.frames, mode == "onehot", _lib.DTYPE_F16 if half else _lib.DTYPE_F32, layout)
        g = self.case.grid
        scratch = None
        if layout == _lib.BEV_NHWC:
            store = torch.zeros((self.frames, g.X, g.Y, C), dtype=torch.float32, device=_dev())
            bev = store.permute(0, 3, 1, 2)
        else:
            store = out if out is not None else torch.empty((self.frames, C, g.X, g.Y), dtype=torch.float32, device=_dev())
            bev = store
            scratch = torch.zeros(int(lib.fiery_lift_scratch_bytes(desc)) // 4, dtype=torch.float32, device=_dev())
        if warp is None:
            rc = lib.fiery_lift_forward(desc, _ptr(head), _ptr(self.a), _ptr(self.b), *self.frustum(), _ptr(store), _ptr(scratch),
                                        _ptr(plan), _stream())
        else:
            theta, copy = warp
            rc = lib.fiery_lift_forward_warped(desc, _ptr(head), _ptr(self.a), _ptr(self.b), *self.frustum(), _ptr(store),
                                               _ptr(scratch), _ptr(plan), _ptr(theta), _ptr(copy), _stream())
        _lib.check(rc, "fiery_lift_forward")
        if scratch is not None:
            assert int(torch.count_nonzero(scratch)) == 0, "the forward left its scratch dirty"
        return bev

    def backward(self, mode, gbev, layout=_lib.BEV_NCHW, plan=None):
        lib = _lib.load()
        head = self.head(mode)[0].to(_dev())
        desc = _desc(self.case, self.frames, mode == "onehot", _lib.DTYPE_F32, layout)
        g = gbev.to(_dev())
        g = g.permute(0, 2, 3, 1).contiguous() if layout == _lib.BEV_NHWC else g.contiguous()
        ws = torch.empty(max(1, int(lib.fiery_lift_workspace_bytes(desc)) // 4), dtype=torch.float32, device=_dev())
        grad = torch.full_like(head, float("nan"))
        _lib.check(lib.fiery_lift_backward(desc, _ptr(head), _ptr(self.a), _ptr(self.b), *self.frustum(), _ptr(g), _ptr(grad),
                                           _ptr(ws), _ptr(plan), _stream()), "fiery_lift_backward")
        return grad


_RUNS = {}


def _run(name, frames):
    key = (name, frames)
    if key not in _RUNS:
        _RUNS[key] = Run(CASES[name] if name in CASES else BIG[name], frames)
    return _RUNS[key]


def _frames_for_dd(case, dd):
    """Frame count whose forward without a plan runs the tile kernel with DD depths per unit (every frame group, both layouts)."""
    tiles = case.n * ((case.u.size + 3) // 4)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    for frames in range(1, 200):
        picks = _unit_kernels(frames, tiles, n_sm, False, False, True) | _unit_kernels(frames, tiles, n_sm, False, False, False)
        if {p[0] for p in picks} == {dd}:
            return frames
    raise AssertionError((case.name, dd))


def _assert_indices(run, idx, valid, pillar):
    assert np.array_equal(valid.astype(bool), run.keep)
    assert np.array_equal(pillar, run.pillar)
    spec = np.isfinite(run.s) & (np.abs(run.s.astype(np.float64)) < G.INT64_EDGE)     # idx_out is specified there only
    assert np.array_equal(idx[spec], run.idx[spec])


def _assert_plan(run, plan):
    dense, tiles, touched = _decode(plan.cpu().numpy(), Shape(run.case, run.frames))
    assert np.array_equal(dense, run.pillar)
    want = np.zeros((run.frames, run.XY), dtype=bool)
    for f in range(run.frames):
        want[f, np.unique(run.pillar[f][run.pillar[f] >= 0])] = True
    assert np.array_equal(touched != 0, want)
    for t in tiles:
        assert_tile_streams(t, run.case.v.size)


# ---- 1. every path, every case -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES), ids=list(CASES))
def test_point_indices_match_the_explicit_chain(name):
    run = _run(name, _frames_for_dd(CASES[name], 3))
    assert run.keep.any() and (~run.keep).any()
    _assert_indices(run, *run.point_indices())


@pytest.mark.parametrize("name", list(CASES), ids=list(CASES))
def test_plan_decodes_to_the_oracle_ranks(name):
    run = _run(name, 2)
    _assert_plan(run, run.plan())


ROUTES = ["dd2", "dd3", "plan"]


@pytest.mark.parametrize("mode", ["onehot", "uniform"])
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("name", list(CASES), ids=list(CASES))
def test_forward_equals_fp64_pooling(name, route, mode):
    """NCHW and NHWC, fp32 and native fp16 heads: the BEV equals fp64 pooling at the oracle's indices exactly."""
    case = CASES[name]
    frames = 2 if route == "plan" else _frames_for_dd(case, int(route[2]))
    run = _run(name, frames)
    want = run.expected_bev(mode)
    plan = run.plan() if route == "plan" else None
    for half in (False, True):
        for layout in (_lib.BEV_NCHW, _lib.BEV_NHWC):
            got = run.forward(mode, half, layout, plan).cpu()
            assert torch.equal(got.double(), want), (half, layout, float((got.double() - want).abs().max()))


@pytest.mark.parametrize("name", list(CASES), ids=list(CASES))
def test_warped_forward_copy_and_integer_shift(name):
    """fiery_lift_forward_warped with every copy flag set equals the plain NCHW forward exactly; on power-of-two grids an
    integer-pixel shift equals the fp64 resampling of the exact BEV."""
    run = _run(name, 2)
    g = run.case.grid
    dev = _dev()
    plan = run.plan()
    for p in (None, plan):
        plain = run.forward("onehot", plan=p)
        theta = torch.tensor([[1.0, 0.0, 0.0, 0.0, 1.0, 0.0]] * run.frames, device=dev).view(run.frames, 2, 3)
        copied = run.forward("onehot", plan=p, warp=(theta, torch.ones(run.frames, dtype=torch.uint8, device=dev)))
        assert torch.equal(copied, plain)
        if (g.X & (g.X - 1)) == 0 and (g.Y & (g.Y - 1)) == 0:
            shift = torch.tensor([[1.0, 0.0, 3 * 2.0 / g.Y, 0.0, 1.0, -2 * 2.0 / g.X]] * run.frames, dtype=torch.float64)
            shift = shift.view(run.frames, 2, 3)
            got = run.forward("onehot", plan=p, warp=(shift.float().to(dev), torch.zeros(run.frames, dtype=torch.uint8, device=dev)))
            want = run.expected_bev("onehot")
            grid = F.affine_grid(shift, list(want.shape), align_corners=False)
            want = F.grid_sample(want, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
            assert torch.equal(got.cpu().double(), want)


@pytest.mark.parametrize("mode", ["onehot", "uniform"])
@pytest.mark.parametrize("name", list(CASES), ids=list(CASES))
def test_backward_equals_fp64_gradient(name, mode):
    run = _run(name, 2)
    g = run.case.grid
    gen = torch.Generator().manual_seed(5)
    gbev = torch.randint(-4, 5, (run.frames, C, g.X, g.Y), generator=gen).float()
    want = run.expected_grad(mode, gbev)
    plan = run.plan()
    for p in (None, plan):
        for layout in (_lib.BEV_NCHW, _lib.BEV_NHWC):
            got = run.backward(mode, gbev, layout, p).cpu()
            assert torch.equal(got.double(), want), (p is None, layout)


def test_cases_run_both_unit_shapes():
    for case in (BOUNDARY["boundary-pow2"], RUNS["runs-h32-alt"]):
        assert _frames_for_dd(case, 2) != _frames_for_dd(case, 3)


# ---- 2. grids above 2^24 cells on one axis -------------------------------------------------------------------------------------
BIG = {f"big-{n}": G.boundary_case(g) for n, g in G.BIG_GRIDS.items()}


@pytest.mark.parametrize("name", list(BIG), ids=list(BIG))
def test_grid_edge_above_2p24_indices_and_plan(name):
    """trunc(s) < X with X = 2^24 + 1: s = 2^24 is kept (float(X) rounds down to 2^24, so s < float(X) dropped it); 2^24 and
    2^24 + 3 are the controls.  The transposed grid checks y."""
    run = _run(name, 2)
    X, Y = run.case.grid.X, run.case.grid.Y
    top = (X - 1) * Y if X > 1 else Y - 1
    if run.case.grid.name in ("x2p24p1", "y2p24p1", "x2p24p3"):
        assert (run.pillar == top).any()                                 # the last cell receives points
    _assert_indices(run, *run.point_indices())
    one = _run(name, 1)
    _assert_plan(one, one.plan())


def test_grid_edge_above_2p24_forward():
    """The forward at X = 2^24 + 1 (4.3 GB of output and as much scratch), without and with a plan."""
    free, _ = torch.cuda.mem_get_info(0)
    if free < 12 * 2 ** 30:
        pytest.skip(f"needs about 12 GB of free device memory, {free / 2 ** 30:.1f} GB free")
    run = _run("big-x2p24p1", 1)
    keys, sums = run.pooled("uniform")
    assert (keys == run.case.grid.X - 1).any()
    out = torch.empty((1, C, run.case.grid.X, 1), dtype=torch.float32, device=_dev())
    for p in (None, run.plan()):
        bev = run.forward("uniform", plan=p, out=out).view(C, -1)
        got = bev[:, keys.to(_dev())].t().cpu().double()
        assert torch.equal(got, sums)
        assert int(torch.count_nonzero(bev)) == int(torch.count_nonzero(sums))      # nothing anywhere else
        del bev
    del out
    torch.cuda.empty_cache()


# ---- 3. compose_camera: LU with partial pivoting -------------------------------------------------------------------------------
PIVOTS = G.pivot_intrinsics()


def test_compose_calibration_is_bit_exact_at_every_pivot_order():
    """fiery_compose_calibration against the explicit LU (every pivot sequence, first-maximum ties, pinholes) wherever the result
    is finite; singular and non-finite intrinsics give a non-finite result there too."""
    Ks = np.stack([K for _, K, _ in PIVOTS]).astype(np.float32)
    Es = G.pivot_extrinsics(len(PIVOTS))
    want_c, want_t = O.compose_calibration_explicit(Ks, Es)
    dev = _dev()
    K, E = torch.from_numpy(Ks).to(dev), torch.from_numpy(Es).to(dev)
    comb = torch.empty((len(PIVOTS), 3, 3), dtype=torch.float32, device=dev)
    trans = torch.empty((len(PIVOTS), 3), dtype=torch.float32, device=dev)
    _lib.check(_lib.load().fiery_compose_calibration(len(PIVOTS), _ptr(K), _ptr(E), _ptr(comb), _ptr(trans), _stream()),
               "fiery_compose_calibration")
    comb, trans = comb.cpu().numpy(), trans.cpu().numpy()
    assert np.array_equal(trans, want_t)
    for i, (name, _, claim) in enumerate(PIVOTS):
        if np.isfinite(want_c[i]).all():
            assert claim != "singular", name
            assert np.array_equal(comb[i].view(np.uint32), want_c[i].view(np.uint32)), (name, comb[i], want_c[i])
        else:
            assert not np.isfinite(comb[i]).all(), name


def test_raw_calibration_paths_match_the_composed_ones():
    """With FIERY_CALIB_RAW every path composes R @ K^-1 itself: point indices, plan, forward and backward equal the same calls
    with the explicit LU's combined passed in, for every pivot case; where the product is not finite every point is masked --
    zero BEV, clean scratch, an all-zero touched map and a zero gradient."""
    case = G.run_case(8, "alt")
    n_cam = len(PIVOTS)
    Ks = np.stack([K for _, K, _ in PIVOTS]).astype(np.float32)
    Es = G.pivot_extrinsics(n_cam)
    comb, trans = O.compose_calibration_explicit(Ks, Es)
    case = G.Case("pivots", case.grid, case.u, np.linspace(-0.8, 0.8, 8).astype(np.float32), np.array([2.0, 6.0, 11.5], np.float32),
                  comb, trans)
    run = Run(case, 1)
    finite = np.isfinite(comb).reshape(n_cam, 9).all(1)
    assert (~finite).sum() >= 5 and finite.sum() >= 10
    raw = Run(case, 1)
    raw.a, raw.b = torch.from_numpy(Ks[None]).to(_dev()), torch.from_numpy(Es[None]).to(_dev())
    lib = _lib.load()
    dev = _dev()
    # point indices
    N = case.d.size * case.v.size * case.u.size
    outs = []
    for r, mode in ((run, _lib.CALIB_COMPOSED), (raw, _lib.CALIB_RAW)):
        pil = torch.empty((1, n_cam * N), dtype=torch.int32, device=dev)
        _lib.check(lib.fiery_lift_point_indices(_desc(case, 1, calib=mode), _ptr(r.a), _ptr(r.b), *r.frustum(), 0, 0, _ptr(pil),
                                                _stream()), "fiery_lift_point_indices")
        outs.append(pil.cpu().numpy().reshape(run.pillar.shape))
    assert np.array_equal(outs[0], run.pillar) and np.array_equal(outs[1], run.pillar)
    assert (run.pillar[0, ~finite] == -1).all() and (run.pillar[0, finite] >= 0).any()
    # plan
    plans = []
    for r, mode in ((run, _lib.CALIB_COMPOSED), (raw, _lib.CALIB_RAW)):
        desc = _desc(case, 1, calib=mode)
        buf = torch.empty(int(lib.fiery_lift_plan_bytes(desc)), dtype=torch.uint8, device=dev)
        _lib.check(lib.fiery_lift_plan(desc, _ptr(r.a), _ptr(r.b), *r.frustum(), _ptr(buf), _stream()), "fiery_lift_plan")
        plans.append(buf)
    _assert_plan(run, plans[0])
    _assert_plan(run, plans[1])
    # forward and backward, raw calibration, with and without the plan
    want = run.expected_bev("uniform")
    gbev = torch.randint(-4, 5, (1, C, case.grid.X, case.grid.Y), generator=torch.Generator().manual_seed(9)).float()
    want_g = run.expected_grad("uniform", gbev)
    for p in (None, plans[1]):
        for layout in (_lib.BEV_NCHW, _lib.BEV_NHWC):
            head = run.head("uniform")[0].to(dev)
            desc = _desc(case, 1, False, _lib.DTYPE_F32, layout, calib=_lib.CALIB_RAW)
            if layout == _lib.BEV_NHWC:
                store = torch.zeros((1, case.grid.X, case.grid.Y, C), device=dev)
                got, scratch = store.permute(0, 3, 1, 2), None
            else:
                store = got = torch.empty((1, C, case.grid.X, case.grid.Y), device=dev)
                scratch = torch.zeros(int(lib.fiery_lift_scratch_bytes(desc)) // 4, device=dev)
            _lib.check(lib.fiery_lift_forward(desc, _ptr(head), _ptr(raw.a), _ptr(raw.b), *raw.frustum(), _ptr(store), _ptr(scratch),
                                              _ptr(p), _stream()), "fiery_lift_forward")
            assert torch.equal(got.cpu().double(), want), (p is None, layout)
            if scratch is not None:
                assert int(torch.count_nonzero(scratch)) == 0
            g = gbev.to(dev)
            g = g.permute(0, 2, 3, 1).contiguous() if layout == _lib.BEV_NHWC else g
            ws = torch.empty(max(1, int(lib.fiery_lift_workspace_bytes(desc)) // 4), device=dev)
            grad = torch.full_like(head, float("nan"))
            _lib.check(lib.fiery_lift_backward(desc, _ptr(head), _ptr(raw.a), _ptr(raw.b), *raw.frustum(), _ptr(g), _ptr(grad),
                                               _ptr(ws), _ptr(p), _stream()), "fiery_lift_backward")
            assert torch.equal(grad.cpu().double(), want_g), (p is None, layout)
            assert float(grad.view(n_cam, -1)[torch.from_numpy(~finite).to(dev)].abs().max()) == 0.0


def test_non_finite_calibration_masks_every_point():
    """Only singular / non-finite intrinsics in the batch: zero BEV, clean scratch, no touched pillar, zero gradient."""
    bad = [(K, claim) for _, K, claim in PIVOTS if claim in ("singular", "nonfinite")]
    Ks = np.stack([K for K, _ in bad]).astype(np.float32)
    Es = G.pivot_extrinsics(len(bad))
    comb, _ = O.compose_calibration_explicit(Ks, Es)
    keep = ~np.isfinite(comb).reshape(len(bad), 9).all(1)
    Ks, Es = Ks[keep], Es[keep]
    base = G.run_case(4, "alt")
    comb, trans = O.compose_calibration_explicit(Ks, Es)
    case = G.Case("masked", base.grid, base.u, base.v, base.d, comb, trans)
    run = Run(case, 1)
    run.a, run.b = torch.from_numpy(Ks[None]).to(_dev()), torch.from_numpy(Es[None]).to(_dev())
    assert (run.pillar == -1).all()
    lib = _lib.load()
    dev = _dev()
    desc = _desc(case, 1, calib=_lib.CALIB_RAW)
    buf = torch.empty(int(lib.fiery_lift_plan_bytes(desc)), dtype=torch.uint8, device=dev)
    _lib.check(lib.fiery_lift_plan(desc, _ptr(run.a), _ptr(run.b), *run.frustum(), _ptr(buf), _stream()), "fiery_lift_plan")
    _assert_plan(run, buf)
    head = run.head("onehot")[0].to(dev)
    for p in (None, buf):
        out = torch.full((1, C, case.grid.X, case.grid.Y), float("nan"), device=dev)
        scratch = torch.zeros(int(lib.fiery_lift_scratch_bytes(desc)) // 4, device=dev)
        _lib.check(lib.fiery_lift_forward(desc, _ptr(head), _ptr(run.a), _ptr(run.b), *run.frustum(), _ptr(out), _ptr(scratch),
                                          _ptr(p), _stream()), "fiery_lift_forward")
        assert int(torch.count_nonzero(out)) == 0 and int(torch.count_nonzero(scratch)) == 0
        g = torch.ones((1, C, case.grid.X, case.grid.Y), device=dev)
        ws = torch.empty(max(1, int(lib.fiery_lift_workspace_bytes(desc)) // 4), device=dev)
        grad = torch.full_like(head, float("nan"))
        _lib.check(lib.fiery_lift_backward(desc, _ptr(head), _ptr(run.a), _ptr(run.b), *run.frustum(), _ptr(g), _ptr(grad), _ptr(ws),
                                           _ptr(p), _stream()), "fiery_lift_backward")
        assert int(torch.count_nonzero(grad)) == 0
