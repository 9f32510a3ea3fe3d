"""GPU: the lift across the shapes its C ABI accepts and the launch routes its launcher can take, against the fp64 oracle.

The limits fiery_lift_forward / _plan / _backward enforce are depth_bins 1..48, feat_h 1..32, feat_w a multiple of 4, any BEV grid,
any camera count, C = 64.  The kernels branch on exactly these values: the depth TMA box is always 48 rows and the softmax masks
the rows past D; the tile kernel's units hold 2 or 3 depths and the plan / backward use groups of 4 depths and 4 row groups (h < 4
leaves row groups empty); the row masks are 32 bits; X*Y % 4 != 0 switches the NCHW layout pass from the TMA kernel to
finalize_nchw_kernel.  The launcher picks the tile kernel's unit shape, cuts a pass into frame groups on two scratch lanes and a
call into passes.  Each route below is checked value for value against oracle.lift_exact (fp64 direct pooling) and the fp64
autograd gradient, with the bars of the other lift tests, and asserts that it actually ran."""
import numpy as np
import pytest
import torch

from fiery_b200 import _lib
from fiery_b200 import lift as lift_mod
from fiery_b200.lift import LiftSplat
from fiery_b200.synthetic import CONFIGS, LiftConfig, make_calibration, make_egomotion, make_grad_bev, make_head
from fiery_b200.warp import cumulative_warp_features
from oracle import lift_oracle as O
from oracle import warp_oracle as W
from tests.test_lift_backward_gpu import _oracle_grad
from tests.test_lift_launch_plan_cpu import forward_groups, group_bounds, passes, scratch_bytes
from tests._plan_layout import PAIRS, _decode

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _dev():
    return torch.device("cuda:0")


# ---- shared checks ------------------------------------------------------------------------------------------------------------
def _assert_bev(got: torch.Tensor, exact: torch.Tensor, what):
    """BEV (B', C, X, Y) against the fp64 pooling: same occupied pillars, empty pillars exactly zero, normwise, max-abs-scaled and
    element-wise relative error (on elements above 1e-2 of the maximum: smaller ones are cancellation results)."""
    got = got.detach().cpu().contiguous()
    assert got.shape == exact.shape and got.dtype == torch.float32, what
    occ = exact.abs().sum(1) > 0
    assert torch.equal(got.abs().sum(1) > 0, occ), what
    if (~occ).any():
        assert float(got.abs().amax(1)[~occ].max()) == 0.0, what
    assert O.normwise_error(got, exact) < TOL, (what, O.normwise_error(got, exact))
    assert O.max_abs_scaled_error(got, exact) < TOL, (what, O.max_abs_scaled_error(got, exact))
    _assert_elementwise(got, exact, what)


def _assert_elementwise(got, exact, what):
    big = exact.abs() > 1e-2 * exact.abs().max()
    rel = ((got.double() - exact).abs() / exact.abs())[big]
    assert float(rel.max()) < TOL, (what, float(rel.max()))


def _assert_grad(got: torch.Tensor, exact: torch.Tensor, what):
    got = got.detach().cpu()
    assert got.shape == exact.shape, what
    assert O.normwise_error(got, exact) < TOL, (what, O.normwise_error(got, exact))
    assert O.max_abs_scaled_error(got, exact) < TOL, (what, O.max_abs_scaled_error(got, exact))
    _assert_elementwise(got, exact, what)


_ORACLE = {}        # (case key, what) -> oracle result, computed once per module run


def _exact(key, cfg, head, K, E):
    """oracle.lift_exact of every frame, one frame at a time (the fp64 volume of a whole batch does not fit comfortably)."""
    if key not in _ORACLE:
        oracle = O.LiftOracle.from_config(cfg)
        n = cfg.n_cameras
        _ORACLE[key] = torch.cat([oracle.lift_exact(head[f * n:(f + 1) * n], K[f:f + 1], E[f:f + 1]) for f in range(K.shape[0])])
    return _ORACLE[key]


def _exact_grad(key, cfg, head, K, E, gout):
    """fp64 autograd gradient of <lift(head), gout> (tests/test_lift_backward_gpu._oracle_grad), one frame at a time."""
    if key not in _ORACLE:
        n = cfg.n_cameras
        _ORACLE[key] = torch.cat([_oracle_grad(cfg, head[f * n:(f + 1) * n], K[f:f + 1], E[f:f + 1], gout[f:f + 1], exact=True)
                                  for f in range(K.shape[0])])
    return _ORACLE[key]


def _launches(lift, frames, n_cameras, layout=_lib.BEV_NCHW):
    c = lift._constants(_dev())
    return int(_lib.load().fiery_lift_forward_launches(lift._desc(c, frames, n_cameras, torch.float32, _lib.CALIB_RAW, layout)))


def _assert_scratch_clean():
    assert lift_mod._scratch._bufs
    for buf in lift_mod._scratch._bufs.values():
        assert float(buf.abs().max()) == 0.0


def _inputs(cfg, seed):
    K, E = make_calibration(cfg, seed=seed)
    return (torch.from_numpy(make_head(cfg, seed=seed)), torch.from_numpy(K), torch.from_numpy(E),
            torch.from_numpy(make_grad_bev(cfg, seed=seed)))


# ---- A. shape sweep ------------------------------------------------------------------------------------------------------------
# final_dim = (8h, 8w); d_bound picks D (ceil((hi - lo) / step) bins); bounds with odd cell counts where X*Y % 4 != 0 is wanted.
SHAPES = {
    # one depth bin: the softmax of a single logit is 1
    "D1-h8-w16-n1": LiftConfig("D1", n_cameras=1, final_dim=(64, 128), x_bound=(-50.0, 50.0, 2.0), y_bound=(-50.0, 50.0, 2.0),
                               d_bound=(20.0, 21.0, 1.0), frames=2),
    # 51 x 49 = 2499 pillars, X*Y % 4 == 3: the fallback layout pass
    "D7-h5-w12-n3-51x49": LiftConfig("D7", n_cameras=3, final_dim=(40, 96), x_bound=(-51.0, 51.0, 2.0), y_bound=(-49.0, 49.0, 2.0),
                                     d_bound=(4.0, 46.0, 6.0), frames=2),
    # h = 32: the last bit of the row masks; 0.4 / 0.3 m cells take the true-division path
    "D17-h32-w20-n2-250x200": LiftConfig("D17", n_cameras=2, final_dim=(256, 160), x_bound=(-50.0, 50.0, 0.4),
                                         y_bound=(-30.0, 30.0, 0.3), d_bound=(2.0, 53.0, 3.0), frames=2),
    # one image row: three of the four row groups of the plan and the backward are empty; 101 x 99 = 9999 pillars (fallback pass)
    "D41-h1-w60-n6-101x99": LiftConfig("D41", n_cameras=6, final_dim=(8, 480), x_bound=(-50.5, 50.5, 1.0), y_bound=(-49.5, 49.5, 1.0),
                                       d_bound=(4.0, 45.0, 1.0), frames=2),
    # one column tile
    "D45-h3-w4-n5": LiftConfig("D45", n_cameras=5, final_dim=(24, 32), x_bound=(-50.0, 50.0, 2.0), y_bound=(-50.0, 50.0, 2.0),
                               d_bound=(2.0, 47.0, 1.0), frames=2),
    "D45-h3-w4-n5-uniform": LiftConfig("D45u", n_cameras=5, final_dim=(24, 32), x_bound=(-50.0, 50.0, 2.0),
                                       y_bound=(-50.0, 50.0, 2.0), d_bound=(2.0, 47.0, 1.0), frames=2, use_depth_distribution=False),
    # D not a multiple of 3, 4 or 8; two rows
    "D47-h2-w36-n6": LiftConfig("D47", n_cameras=6, final_dim=(16, 288), d_bound=(2.0, 49.0, 1.0), frames=2),
    # odd row count at full depth
    "D48-h31-w36-n6": LiftConfig("D48", n_cameras=6, final_dim=(248, 288), d_bound=(2.0, 50.0, 1.0), frames=2),
}
SHAPE_WANT = {"D1-h8-w16-n1": (1, 8, 16, (50, 50)), "D7-h5-w12-n3-51x49": (7, 5, 12, (51, 49)),
              "D17-h32-w20-n2-250x200": (17, 32, 20, (250, 200)), "D41-h1-w60-n6-101x99": (41, 1, 60, (101, 99)),
              "D45-h3-w4-n5": (45, 3, 4, (50, 50)), "D45-h3-w4-n5-uniform": (45, 3, 4, (50, 50)),
              "D47-h2-w36-n6": (47, 2, 36, (200, 200)), "D48-h31-w36-n6": (48, 31, 36, (200, 200))}
# at least this many valid frustum points and occupied pillars in every frame: a calibration that missed the grid would pass trivially
MIN_POINTS, MIN_PILLARS = 100, 10


@pytest.fixture(scope="module", params=list(SHAPES), ids=list(SHAPES))
def shape(request):
    name = request.param
    cfg = SHAPES[name]
    D, h, w, bev = SHAPE_WANT[name]
    assert (cfg.depth_bins, *cfg.feat_hw, cfg.bev_hw) == (D, h, w, bev)
    head, K, E, gout = _inputs(cfg, seed=7 + list(SHAPES).index(name))
    dev = _dev()
    return dict(name=name, cfg=cfg, head=head, K=K, E=E, gout=gout, hd=head.to(dev), Kd=K.to(dev), Ed=E.to(dev), gd=gout.to(dev))


def test_shape_case_is_not_vacuous(shape):
    cfg, K, E = shape["cfg"], shape["K"], shape["E"]
    _, keep = O.LiftOracle.from_config(cfg).point_indices(K, E)
    exact = _exact((shape["name"], "bev"), cfg, shape["head"], K, E)
    for f in range(cfg.frames):
        assert int(keep[f].sum()) >= MIN_POINTS, (f, int(keep[f].sum()))
        assert int((exact[f].abs().sum(0) > 0).sum()) >= MIN_PILLARS, f
    assert (np.prod(cfg.bev_hw) % 4 != 0) == shape["name"].endswith(("51x49", "101x99"))


@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
def test_shape_forward_matches_oracle(shape, layout):
    cfg = shape["cfg"]
    lift = LiftSplat.from_config(cfg, output_layout=layout).to(_dev())
    exact = _exact((shape["name"], "bev"), cfg, shape["head"], shape["K"], shape["E"])
    with torch.no_grad():
        for p in (None, lift.plan(shape["Kd"], shape["Ed"])):
            for _ in range(2):                                        # the second call finds the scratch the first one left
                bev = lift(shape["hd"], shape["Kd"], shape["Ed"], plan=p)
            _assert_bev(bev, exact, (layout, p is None))
    if layout == "contiguous":
        assert bev.is_contiguous()
        _assert_scratch_clean()


def test_shape_plan_decodes_to_oracle_ranks(shape):
    """The plan, decoded to one pillar per frustum point, equals the oracle's ranks (fiery.py:236-256); its touched map is the set of
    pillars that receive a point; its run lists are tight."""
    cfg, K, E = shape["cfg"], shape["K"], shape["E"]
    lift = LiftSplat.from_config(cfg).to(_dev())
    plan = lift.plan(shape["Kd"], shape["Ed"])
    dense, tiles, touched = _decode(plan.cpu().numpy(), cfg)
    h, w = cfg.feat_hw
    X, Y = cfg.bev_hw
    idx, keep = O.LiftOracle.from_config(cfg).point_indices(K, E)
    rank = torch.where(keep, idx[..., 0] * Y + idx[..., 1], torch.full_like(idx[..., 0], -1))
    rank = rank.view(cfg.frames, cfg.n_cameras, cfg.depth_bins, h, w).numpy().astype(np.int32)
    assert np.array_equal(dense, rank)
    want = np.zeros((cfg.frames, X * Y), dtype=np.uint8)
    for f in range(cfg.frames):
        want[f, np.unique(rank[f][rank[f] >= 0])] = 1
    assert np.array_equal(touched != 0, want != 0)
    for t in tiles:
        assert t["n_runs"] == PAIRS + sum(bin(int(m)).count("1") for m in t["mask"])


@pytest.mark.parametrize("grad_layout", ["contiguous", "channels_last"])
def test_shape_backward_matches_fp64_gradient(shape, grad_layout):
    cfg = shape["cfg"]
    lift = LiftSplat.from_config(cfg).to(_dev())
    exact = _exact_grad((shape["name"], "grad"), cfg, shape["head"], shape["K"], shape["E"], shape["gout"])
    g = shape["gd"]
    if grad_layout == "channels_last":
        g = g.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    hd = shape["hd"].clone().requires_grad_(True)
    lift(hd, shape["Kd"], shape["Ed"]).backward(g)                   # the autograd path: one plan for forward and backward
    _assert_grad(hd.grad, exact, "autograd")
    _assert_grad(lift._launch_backward(shape["hd"], shape["Kd"], shape["Ed"], g, plan=None), exact, "no plan")


@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
def test_shape_native_fp16_head(shape, layout):
    """The tile kernel reading the fp16 head itself (NATIVE_FP16_FORWARD) against the exact lift of the widened values."""
    cfg = shape["cfg"]
    h16 = shape["hd"].half()
    exact = _exact((shape["name"], "f16"), cfg, h16.float().cpu(), shape["K"], shape["E"])
    lift = LiftSplat.from_config(cfg, output_layout=layout).to(_dev())
    old = lift_mod.NATIVE_FP16_FORWARD
    lift_mod.NATIVE_FP16_FORWARD = True
    try:
        with torch.no_grad():
            for p in (None, lift.plan(shape["Kd"], shape["Ed"])):
                _assert_bev(lift._launch_forward(h16, shape["Kd"], shape["Ed"], plan=p), exact, p is None)
    finally:
        lift_mod.NATIVE_FP16_FORWARD = old


# ---- B. unit shape of the tile kernel ------------------------------------------------------------------------------------------
# Mirror of launch_forward_cols (fiery_b200/csrc/lift_fwd_cols.cu): every launch -- one per frame group -- picks DD = 3 depths per
# unit when it has a plan, or when its tiles fill whole waves of 2 tiles per SM or leave a last wave more than half full
# (n_tiles % (2 * n_sm) == 0 or > n_sm); DD = 2 otherwise.  Each comes with an fp32 or an fp16 head, and with NCHW output (L2
# hints, reducing into the scratch) or channel-last output: 8 kernels without a plan and 4 with one.
UNIT_CFG = LiftConfig("unit", n_cameras=6, final_dim=(64, 480), frames=1)      # 90 tiles per frame, D = 48, h = 8


def _unit_kernels(frames, tiles_per_frame, n_sm, planned, half, nchw):
    """The tile kernels one forward call launches (no forced pass cap: the call is one pass)."""
    out = set()
    for s0, s1 in group_bounds(frames, forward_groups(frames, tiles_per_frame, nchw)):
        rem = (s1 - s0) * tiles_per_frame % (2 * n_sm)
        dd = 3 if planned or not (0 < rem <= n_sm) else 2
        out.add((dd, "f16" if half else "f32", "nchw" if nchw else "nhwc", "plan" if planned else "geometry"))
    return out


UNIT_PICKS = [(dd, dt, lay, how, frames)
              for dd, how, frames in ((2, "geometry", 1), (3, "geometry", 2), (3, "plan", 1))
              for dt in ("f32", "f16") for lay in ("nchw", "nhwc")]


@pytest.mark.parametrize("dd,dtype,layout,how,frames", UNIT_PICKS, ids=["-".join(map(str, p)) for p in UNIT_PICKS])
def test_every_tile_kernel_unit_shape_matches_oracle(dd, dtype, layout, how, frames):
    cfg = LiftConfig(**{**UNIT_CFG.__dict__, "frames": frames})
    tiles = cfg.n_cameras * ((cfg.feat_hw[1] + 3) // 4)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    want = (dd, dtype, layout, how)
    assert _unit_kernels(frames, tiles, n_sm, how == "plan", dtype == "f16", layout == "nchw") == {want}, (want, n_sm)
    head, K, E, _ = _inputs(cfg, seed=70 + frames)
    dev = _dev()
    hd, Kd, Ed = head.to(dev), K.to(dev), E.to(dev)
    lift = LiftSplat.from_config(cfg, output_layout="contiguous" if layout == "nchw" else "channels_last").to(dev)
    plan = lift.plan(Kd, Ed) if how == "plan" else None
    if dtype == "f16":
        hd = hd.half()
        head = hd.float().cpu()
    exact = _exact(("unit", frames, dtype), cfg, head, K, E)
    old = lift_mod.NATIVE_FP16_FORWARD
    lift_mod.NATIVE_FP16_FORWARD = dtype == "f16"
    try:
        with torch.no_grad():
            _assert_bev(lift._launch_forward(hd, Kd, Ed, plan=plan), exact, want)
    finally:
        lift_mod.NATIVE_FP16_FORWARD = old


def test_unit_picks_cover_all_reachable_kernels():
    assert len({p[:4] for p in UNIT_PICKS}) == 12


# ---- C. frame groups, scratch lanes and passes ---------------------------------------------------------------------------------
# Each case runs at least 3 frame groups, so a lane reduces a second group into the slice its first group's layout pass restored.
# 90 tiles per frame, D = 12, h = 8: cheap for the oracle, and 8 frames are 4 groups of 2 frames
ROUTE_TMA = LiftConfig("route_tma", n_cameras=6, final_dim=(64, 480), d_bound=(2.0, 50.0, 4.0))
# 201 x 199 = 39999 pillars: not a multiple of 4 (fallback layout pass) nor of 64 (the warped layout pass's last tile is partial)
ROUTE_ODD = LiftConfig("route_odd", n_cameras=6, final_dim=(64, 480), d_bound=(2.0, 50.0, 4.0), x_bound=(-50.25, 50.25, 0.5),
                       y_bound=(-49.75, 49.75, 0.5))


def _frames(cfg, frames):
    return LiftConfig(**{**cfg.__dict__, "frames": frames})


def _warped_case(base, b, s, seed, plan):
    cfg = _frames(base, b * s)
    head, K, E, _ = _inputs(cfg, seed)
    flow = torch.from_numpy(make_egomotion(b, s, seed=seed))
    ext = (float(cfg.x_bound[1]), float(cfg.y_bound[1]))
    dev = _dev()
    hd, Kd, Ed, fd = head.to(dev), K.to(dev), E.to(dev), flow.to(dev)
    lift = LiftSplat.from_config(cfg).to(dev)
    assert _launches(lift, b * s, cfg.n_cameras) >= 2 * 3
    p = lift.plan(Kd, Ed) if plan else None
    with torch.no_grad():
        first = lift.forward_warped(hd, Kd, Ed, fd, ext, plan=p)
        fused = lift.forward_warped(hd, Kd, Ed, fd, ext, plan=p)      # the scratch the first call left must be clean
        unfused = cumulative_warp_features(lift(hd, Kd, Ed).unflatten(0, (b, s)), fd, mode="bilinear", spatial_extent=ext)
    _assert_scratch_clean()
    scale = float(unfused.abs().max())
    assert float((fused - first).abs().max()) <= 5e-6 * scale
    assert float((fused - unfused).abs().max()) <= 5e-6 * scale       # same samples, same blend; only the lift's atomics differ
    exact = _exact((base.name, b, s, seed), cfg, head, K, E).unflatten(0, (b, s))
    want = W.cumulative_warp_features(exact.clone().float(), flow, mode="bilinear", spatial_extent=ext)
    assert float((fused.cpu() - want).abs().max()) <= TOL * float(want.abs().max())
    assert O.normwise_error(fused.cpu(), want) < TOL


@pytest.mark.parametrize("plan", [False, True], ids=["geometry", "plan"])
def test_warped_forward_over_four_frame_groups(plan):
    """fiery_lift_forward_warped at cfg3_baseline, b = 2, s = 4: 8 frames in 4 groups on 2 lanes (finalize_warp_kernel +
    clear_touched_kernel restore a slice the lane's next group reduces into)."""
    _warped_case(CONFIGS["cfg3_baseline"], 2, 4, seed=81, plan=plan)


@pytest.mark.parametrize("plan", [False, True], ids=["geometry", "plan"])
def test_warped_forward_partial_last_tile(plan):
    assert np.prod(ROUTE_ODD.bev_hw) % 64 != 0
    _warped_case(ROUTE_ODD, 2, 4, seed=82, plan=plan)


def _run_frames(cfg, plan, calls=2):
    """`calls` forward calls of the whole batch (NCHW); every frame against the oracle, the scratch clean afterwards."""
    head, K, E, _ = _inputs(cfg, seed=90 + cfg.frames)
    dev = _dev()
    hd, Kd, Ed = head.to(dev), K.to(dev), E.to(dev)
    lift = LiftSplat.from_config(cfg).to(dev)
    p = lift.plan(Kd, Ed) if plan else None
    with torch.no_grad():
        for _ in range(calls):
            bev = lift(hd, Kd, Ed, plan=p).cpu()
    _assert_scratch_clean()
    exact = _exact((cfg.name, cfg.frames), cfg, head, K, E)
    for f in range(cfg.frames):
        _assert_bev(bev[f:f + 1], exact[f:f + 1], (cfg.name, f, plan))
    return lift


def test_planned_forward_reuses_slices_frame_by_frame():
    """The planned forward's BEV at cfg2_static_lss, 8 frames: 4 groups, so each lane's slice is reused."""
    cfg = _frames(CONFIGS["cfg2_static_lss"], 8)
    lift = _run_frames(cfg, plan=True)
    assert _launches(lift, 8, cfg.n_cameras) == 2 * 4


@pytest.mark.parametrize("plan", [False, True], ids=["geometry", "plan"])
def test_fallback_layout_pass_over_frame_groups(plan):
    cfg = _frames(ROUTE_ODD, 8)
    assert np.prod(cfg.bev_hw) % 4 != 0                  # finalize_nchw_kernel, not the TMA layout pass
    lift = _run_frames(cfg, plan)
    assert _launches(lift, 8, cfg.n_cameras) == 2 * 4


@pytest.mark.parametrize("plan", [False, True], ids=["geometry", "plan"])
@pytest.mark.parametrize("base", [ROUTE_TMA, ROUTE_ODD], ids=["tma", "fallback"])
def test_tail_pass_larger_than_a_full_pass(base, plan):
    """Passes capped at 8 of 15 frames (test hook): the full pass is 4 groups of 2 frames (4 scratch frames), the 7-frame tail 3
    groups of 2, 2 and 3 frames -- 5 scratch frames, so the scratch is sized by the tail."""
    cfg = _frames(base, 15)
    lib = _lib.load()
    pillars = int(np.prod(cfg.bev_hw))
    assert (pillars % 4 == 0) == (base is ROUTE_TMA)
    lib.fiery_lift_set_max_chunk_frames(8)
    try:
        lift_mod._scratch.clear()
        lift = LiftSplat.from_config(cfg).to(_dev())
        c = lift._constants(_dev())
        desc = lift._desc(c, 15, cfg.n_cameras, torch.float32, _lib.CALIB_RAW, _lib.BEV_NCHW)
        assert [nf for _, nf in passes(15, 8)] == [8, 7]
        assert int(lib.fiery_lift_scratch_bytes(desc)) == scratch_bytes(5, pillars)
        assert int(lib.fiery_lift_forward_launches(desc)) == 2 * (4 + 3)
        _run_frames(cfg, plan)
    finally:
        lib.fiery_lift_set_max_chunk_frames(0)
        lift_mod._scratch.clear()
