"""GPU: the geometry plan (fiery_lift_plan, fiery_b200/csrc/lift_plan.cu) -- get_geometry + voxel index / mask / rank of every
frustum point (fiery/models/fiery.py:193-208,236-256) reduced to pillar runs -- is bit-exact: decoded back to one pillar per point
it equals the oracle's ranks; its backward streams and touched map follow from the same runs; and the forward / backward give
the same results with a caller-owned plan, with the plan computed inside the call, and on the multi-pass path."""
import numpy as np
import pytest
import torch

from fiery_b200 import _lib
from fiery_b200.geometry import _stream_ptr
from fiery_b200.lift import LiftSplat
from fiery_b200.synthetic import CONFIGS, LiftConfig, make_calibration, make_grad_bev, make_head
from oracle import lift_oracle as O
from tests._cases import GOLDEN_CASES, build_case, case_id, golden_tag
from tests._plan_layout import TILE_BYTES, _decode, assert_tile_streams

pytestmark = pytest.mark.gpu

@pytest.mark.parametrize("case", GOLDEN_CASES, ids=case_id)
def test_plan_decodes_to_the_reference_ranks(golden_lift, case):
    cfg, K, E, _, _ = build_case(case)
    dev = torch.device("cuda:0")
    lift = LiftSplat.from_config(cfg).to(dev)
    lib = _lib.load()
    plan = lift.plan(K.to(dev), E.to(dev))
    c = lift._constants(dev)
    desc = lift._desc(c, cfg.frames, cfg.n_cameras, torch.float32, _lib.CALIB_RAW, _lib.BEV_NCHW)
    h, w = cfg.feat_hw
    n_tiles = cfg.frames * cfg.n_cameras * ((w + 3) // 4)
    X, Y = cfg.bev_hw
    assert int(lib.fiery_lift_plan_bytes(desc)) == n_tiles * TILE_BYTES + (cfg.frames * X * Y + 127) // 128 * 128 == plan.numel()
    dense, tiles, touched = _decode(plan.cpu().numpy(), cfg)
    # the oracle's ranks (fiery.py:236-256), with the reference-recorded calibration product
    oracle = O.LiftOracle.from_config(cfg)
    comb = torch.from_numpy(golden_lift[f"{golden_tag(case)}__combined"])
    idx, keep = oracle.point_indices(K, E, combined=comb)
    rank = torch.where(keep, idx[..., 0] * Y + idx[..., 1], torch.full_like(idx[..., 0], -1))
    rank = rank.view(cfg.frames, cfg.n_cameras, cfg.depth_bins, h, w).numpy().astype(np.int32)
    assert np.array_equal(dense, rank)
    # touched map == set of pillars that receive a point
    want = np.zeros((cfg.frames, X * Y), dtype=np.uint8)
    for f in range(cfg.frames):
        r = rank[f][rank[f] >= 0]
        want[f, np.unique(r)] = 1
    assert np.array_equal(touched != 0, want != 0)
    # run lists are tight and the backward streams list, per (row group, column, slot), the run containing the group's first row
    # followed by the runs that start inside the group, depth group after depth group, then two pads
    for t in tiles[:: max(1, len(tiles) // 7)]:
        assert_tile_streams(t, h)


@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
def test_caller_owned_plan_matches_internal_plan(layout):
    """Forward and backward with a plan from LiftSplat.plan() equal the calls that compute the geometry themselves; the plan is
    read only (a second call gives the same result) and the scratch invariant holds."""
    cfg = LiftConfig(**{**CONFIGS["cfg2_static_lss"].__dict__, "frames": 5})
    dev = torch.device("cuda:0")
    K, E = make_calibration(cfg, seed=51)
    Kd, Ed = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
    hd = torch.from_numpy(make_head(cfg, seed=51)).to(dev)
    gout = torch.from_numpy(make_grad_bev(cfg, seed=51)).to(dev)
    lift = LiftSplat.from_config(cfg, output_layout=layout).to(dev)
    plan = lift.plan(Kd, Ed)
    snapshot = plan.clone()
    with torch.no_grad():
        internal = lift(hd, Kd, Ed)
        a = lift(hd, Kd, Ed, plan=plan)
        b = lift(hd, Kd, Ed, plan=plan)
    assert O.normwise_error(a.cpu(), internal.cpu()) < 1e-6 and O.normwise_error(b.cpu(), internal.cpu()) < 1e-6
    assert torch.equal(plan, snapshot)
    exact = O.LiftOracle.from_config(cfg).lift_exact(hd.cpu(), torch.from_numpy(K), torch.from_numpy(E))
    assert O.normwise_error(a.cpu().contiguous(), exact) < 1e-4
    # backward: the autograd path makes its own plan; compare with the explicit launches with / without one
    h1 = hd.clone().requires_grad_(True)
    lift(h1, Kd, Ed).backward(gout)
    g_plan = lift._launch_backward(hd, Kd, Ed, gout, plan=plan)
    g_none = lift._launch_backward(hd, Kd, Ed, gout, plan=None)
    assert O.normwise_error(g_plan.cpu(), h1.grad.cpu()) < 1e-6 and O.normwise_error(g_none.cpu(), h1.grad.cpu()) < 1e-6
    with pytest.raises(ValueError):
        small = LiftConfig(**{**cfg.__dict__, "frames": 2})
        k2, e2 = make_calibration(small, seed=1)
        lift(hd, Kd, Ed, plan=lift.plan(torch.from_numpy(k2).to(dev), torch.from_numpy(e2).to(dev)))


def test_static_calibration_capture():
    """LiftSplat.capture(static_calibration=True): the plan is computed once, the replay has no plan kernels."""
    cfg = LiftConfig(**{**CONFIGS["cfg2_static_lss"].__dict__, "frames": 4})
    dev = torch.device("cuda:0")
    K, E = make_calibration(cfg, seed=52)
    Kd, Ed = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
    hd = torch.from_numpy(make_head(cfg, seed=52)).to(dev)
    lift = LiftSplat.from_config(cfg).to(dev)
    with torch.no_grad():
        eager = lift(hd, Kd, Ed).clone()
    g = lift.capture(hd, Kd, Ed, static_calibration=True)
    assert g.plan is not None
    for _ in range(3):
        out = g()
    torch.cuda.synchronize()
    assert O.normwise_error(out.cpu(), eager.cpu()) < 1e-6
    hd.mul_(0.5)                                            # new head values, same calibration: the replay follows
    out2 = g().clone()
    with torch.no_grad():
        assert O.normwise_error(out2.cpu(), lift(hd, Kd, Ed).cpu()) < 1e-6


@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
def test_multi_pass_path_matches_oracle(layout):
    """Batches whose scratch would exceed 1 GiB run in several passes over the same scratch (lift_fwd.cu: the chunk loop).  The
    test hook caps a pass at 4 frames, so 9 frames take passes of 4, 4 and 1 -- each with its own frame groups and layout
    passes -- and must give, in ONE call, the oracle's result for every frame; with the geometry evaluated in the tile kernels and
    with a caller-owned plan of the whole batch."""
    cfg = LiftConfig(**{**CONFIGS["cfg2_static_lss"].__dict__, "frames": 9})
    dev = torch.device("cuda:0")
    K, E = make_calibration(cfg, seed=61)
    Kd, Ed = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
    head = torch.from_numpy(make_head(cfg, seed=61))
    hd = head.to(dev)
    lift = LiftSplat.from_config(cfg, output_layout=layout).to(dev)
    lib = _lib.load()
    oracle = O.LiftOracle.from_config(cfg)
    n = cfg.n_cameras
    with torch.no_grad():
        exact = torch.cat([oracle.lift_exact(head[f * n:(f + 1) * n], torch.from_numpy(K[f:f + 1]), torch.from_numpy(E[f:f + 1]))
                           for f in range(cfg.frames)])
        whole = lift(hd, Kd, Ed).cpu().contiguous()
    plan = lift.plan(Kd, Ed)
    c = lift._constants(dev)
    desc = lift._desc(c, cfg.frames, n, torch.float32, _lib.CALIB_RAW, _lib.BEV_NHWC if layout == "channels_last" else _lib.BEV_NCHW)
    full = int(lib.fiery_lift_scratch_bytes(desc))
    lib.fiery_lift_set_max_chunk_frames(4)
    try:
        from fiery_b200 import lift as lift_mod
        lift_mod._scratch.clear()
        assert int(lib.fiery_lift_scratch_bytes(desc)) < full or layout == "channels_last"
        groups_per_pass = 2 if layout == "contiguous" else 1         # 4 frames = 360 tiles: two chains of >= 132 tiles
        per_group = 2 if layout == "contiguous" else 1
        assert int(lib.fiery_lift_forward_launches(desc)) == (2 * groups_per_pass + 1) * per_group
        with torch.no_grad():
            for p in (None, plan):
                for _ in range(2):                                   # second call: the scratch left by the first must be clean
                    got = lift(hd, Kd, Ed, plan=p).cpu().contiguous()
                for f in range(cfg.frames):
                    assert O.normwise_error(got[f:f + 1], exact[f:f + 1]) < 1e-4, (f, p is None)
                    assert O.max_abs_scaled_error(got[f:f + 1], exact[f:f + 1]) < 1e-4, (f, p is None)
                assert O.normwise_error(got, whole) < 1e-6
        for buf in lift_mod._scratch._bufs.values():
            assert float(buf.abs().max()) == 0.0
    finally:
        lib.fiery_lift_set_max_chunk_frames(0)
        from fiery_b200 import lift as lift_mod
        lift_mod._scratch.clear()
