"""GPU parity tests of the fused lift, through the C ABI (fiery_b200/_lib.py -> libfiery_b200.so).

Bar (BASELINE.json north_star): bit-exact integer rank/geometry indices; BEV features within 1e-4 relative fp32.
The reference's own cumsum path is noisier than 1e-4 element-wise (SURVEY.md section 7, hard part 1), so values are
compared normwise / max-abs-scaled against the oracle AND against the fp64 exact pooling.
"""
import os

import numpy as np
import pytest
import torch

from fiery_b200.lift import LiftSplat
from fiery_b200.synthetic import CONFIGS, LiftConfig, make_calibration, make_head
from oracle import lift_oracle as O
from tests._cases import GOLDEN_CASES, build_case, case_id, golden_str, golden_tag, sha

pytestmark = pytest.mark.gpu
TOL = 1e-4      # north_star: "within 1e-4 relative fp32 on the BEV features"


def _dev():
    return torch.device("cuda:0")


@pytest.mark.parametrize("case", GOLDEN_CASES, ids=case_id)
def test_point_indices_bit_exact(golden_lift, case):
    """(ix, iy, iz), validity and rank of every frustum point equal the reference's (fiery.py:236-256) bit for bit."""
    cfg, K, E, _, _ = build_case(case)
    tag = golden_tag(case)
    lift = LiftSplat.from_config(cfg, calibration="torch").to(_dev())
    oracle = O.LiftOracle.from_config(cfg)
    comb = torch.from_numpy(golden_lift[f"{tag}__combined"])
    idx_o, keep_o = oracle.point_indices(K, E, combined=comb)
    # feed the kernel the same combined matrices the oracle used (pre-composed mode)
    lib_idx, lib_valid, lib_pillar = _indices_composed(lift, comb, torch.from_numpy(golden_lift[f"{tag}__translation"]))
    assert torch.equal(lib_idx.cpu(), idx_o)
    assert torch.equal(lib_valid.cpu(), keep_o)
    X, Y = cfg.bev_hw
    rank_o = torch.where(keep_o, idx_o[..., 0] * Y + idx_o[..., 1], torch.full_like(idx_o[..., 0], -1))
    assert torch.equal(lib_pillar.cpu().long(), rank_o)
    assert sha(lib_idx.cpu().numpy()) == golden_str(golden_lift[f"{tag}__idx_sha256"])       # the reference's own bytes
    assert sha(lib_valid.cpu().numpy()) == golden_str(golden_lift[f"{tag}__keep_sha256"])


def _indices_composed(lift, comb, trans):
    """point_indices with pre-composed calibration: go through the C ABI directly."""
    from fiery_b200 import _lib
    from fiery_b200.geometry import _stream_ptr
    lib = _lib.load()
    dev = _dev()
    c = lift._constants(dev)
    B, n = comb.shape[:2]
    desc = lift._desc(c, B, n, torch.float32, _lib.CALIB_COMPOSED, _lib.BEV_NCHW)
    N = n * c["D"] * c["h"] * c["w"]
    a, b = comb.to(dev).contiguous(), trans.to(dev).contiguous()
    idx = torch.empty((B, N, 3), dtype=torch.int64, device=dev)
    valid = torch.empty((B, N), dtype=torch.uint8, device=dev)
    pillar = torch.empty((B, N), dtype=torch.int32, device=dev)
    _lib.check(lib.fiery_lift_point_indices(desc, a.data_ptr(), b.data_ptr(), c["u"].data_ptr(), c["v"].data_ptr(),
                                            c["d"].data_ptr(), idx.data_ptr(), valid.data_ptr(), pillar.data_ptr(),
                                            _stream_ptr(dev)), "fiery_lift_point_indices")
    return idx, valid.bool(), pillar


@pytest.mark.parametrize("case", GOLDEN_CASES, ids=case_id)
def test_fused_calibration_bit_exact(golden_lift, case):
    """The in-kernel R @ inverse(K) equals the reference's torch result for pinhole intrinsics, and the explicit oracle."""
    cfg, K, E, _, _ = build_case(case)
    lift = LiftSplat.from_config(cfg).to(_dev())
    comb, trans = lift.compose_calibration(K.to(_dev()), E.to(_dev()))
    ce, te = O.compose_calibration_explicit(K.numpy(), E.numpy())
    assert np.array_equal(comb.cpu().numpy(), ce) and np.array_equal(trans.cpu().numpy(), te)
    assert np.array_equal(comb.cpu().numpy(), golden_lift[f"{golden_tag(case)}__combined"])
    # and the default (fused, raw calibration) index path gives the same integers as the pre-composed one
    idx, valid, pillar = lift.point_indices(K.to(_dev()), E.to(_dev()))
    assert sha(idx.cpu().numpy()) == golden_str(golden_lift[f"{golden_tag(case)}__idx_sha256"])


def test_general_intrinsics_close():
    """Non-pinhole K: LU+solve agrees with torch.inverse to a few ulp (documented limit of bit-exactness)."""
    rng = np.random.default_rng(0)
    K = torch.from_numpy(rng.standard_normal((2, 6, 3, 3)).astype(np.float32) + 3 * np.eye(3, dtype=np.float32))
    E = torch.eye(4).repeat(2, 6, 1, 1)
    E[..., :3, :3] = torch.from_numpy(rng.standard_normal((2, 6, 3, 3)).astype(np.float32))
    lift = LiftSplat.from_config(CONFIGS["cfg1_tiny"]).to(_dev())
    comb, _ = lift.compose_calibration(K.to(_dev()), E.to(_dev()))
    ref, _ = O.compose_calibration(K, E)
    assert torch.allclose(comb.cpu(), ref, rtol=2e-5, atol=1e-6)
    ce, _ = O.compose_calibration_explicit(K.numpy(), E.numpy())
    assert np.array_equal(comb.cpu().numpy(), ce)          # the device code and its numpy restatement agree exactly


@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
@pytest.mark.parametrize("case", GOLDEN_CASES, ids=case_id)
def test_forward_matches_oracle(golden_lift, case, layout):
    cfg, K, E, head, _ = build_case(case)
    tag = golden_tag(case)
    dev = _dev()
    lift = LiftSplat.from_config(cfg, output_layout=layout).to(dev)
    bev = lift(head.to(dev), K.to(dev), E.to(dev))
    torch.cuda.synchronize()
    X, Y = cfg.bev_hw
    assert tuple(bev.shape) == (cfg.frames, cfg.out_channels, X, Y) and bev.dtype == torch.float32
    if layout == "contiguous":
        assert bev.is_contiguous()
    got = bev.cpu().contiguous()

    oracle = O.LiftOracle.from_config(cfg)
    comb = torch.from_numpy(golden_lift[f"{tag}__combined"])
    ref = oracle.lift(head, K, E, combined=comb)                    # the reference's cumsum path (O1)
    exact = oracle.lift_exact(head, K, E, combined=comb)            # fp64 direct pooling (O3)
    # same pillars occupied, empty pillars exactly zero (fiery.py:263)
    occ_ref = exact.abs().sum(1) > 0
    assert torch.equal(got.abs().sum(1) > 0, occ_ref)
    assert float(got[~occ_ref.unsqueeze(1).expand_as(got)].abs().max() if (~occ_ref).any() else 0.0) == 0.0
    # values: normwise and max-abs-scaled against both oracles; ours must be the closer one to the fp64 truth
    e_ref, e_ours = O.normwise_error(ref, exact), O.normwise_error(got, exact)
    assert O.normwise_error(got, ref) < TOL and O.max_abs_scaled_error(got, ref) < TOL
    assert e_ours < TOL and O.max_abs_scaled_error(got, exact) < TOL
    assert e_ours <= max(e_ref, 2e-6), (e_ours, e_ref)
    # element-wise relative check against the exact pooling on the well-conditioned elements (a pillar sums up to 420
    # signed products, so tiny values are cancellation results whose relative error is unbounded in any fp32 scheme)
    big = exact.abs() > 1e-2 * exact.abs().max()
    rel = ((got.double() - exact).abs() / exact.abs())[big]
    assert float(rel.max()) < TOL
    # the reference's own recorded bytes (golden): sampled values within the reference's own noise of the exact ones
    pick = golden_lift[f"{tag}__bev_pick"]
    rec = golden_lift[f"{tag}__bev_ref_at_pick"]
    assert np.abs(got.flatten()[pick].numpy() - rec).max() <= TOL * float(np.abs(rec).max())
    assert np.allclose(got.double().flatten(1).norm(dim=1).numpy(), golden_lift[f"{tag}__exact_norm"], rtol=1e-5)


def test_scratch_invariant_and_repeatability():
    """The accumulation scratch is all-zero after a call, so calls can be repeated; results differ only by atomic order."""
    from fiery_b200 import lift as lift_mod
    cfg = LiftConfig(**{**CONFIGS["cfg2_static_lss"].__dict__, "frames": 2})
    dev = _dev()
    K, E = make_calibration(cfg, seed=1)
    head = torch.from_numpy(make_head(cfg, seed=1)).to(dev)
    lift = LiftSplat.from_config(cfg).to(dev)
    a = lift(head, torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev))
    torch.cuda.synchronize()
    assert lift_mod._scratch._bufs
    for buf in lift_mod._scratch._bufs.values():
        assert float(buf.abs().max()) == 0.0
    b = lift(head, torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev))
    assert O.normwise_error(a.cpu(), b.cpu()) < 1e-6


def test_uniform_depth_branch():
    """USE_DEPTH_DISTRIBUTION False: every depth bin receives the context vector (encoder.py:101-102)."""
    base = CONFIGS["cfg1_tiny"]
    cfg = LiftConfig(**{**base.__dict__, "use_depth_distribution": False})
    dev = _dev()
    K, E = make_calibration(cfg, seed=2)
    head = torch.from_numpy(make_head(cfg, seed=2))
    lift = LiftSplat.from_config(cfg).to(dev)
    got = lift(head.to(dev), torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)).cpu()
    oracle = O.LiftOracle.from_config(cfg)
    exact = oracle.lift_exact(head, torch.from_numpy(K), torch.from_numpy(E))
    assert O.normwise_error(got, exact) < TOL and O.max_abs_scaled_error(got, exact) < TOL


def test_linearity_in_context_full_size():
    """Size-independent property at the full benchmark size: the lift is linear in the context channels for fixed
    depth logits, lift(a*ctx1 + ctx2) == a*lift(ctx1) + lift(ctx2)."""
    cfg = CONFIGS["cfg3_baseline"]
    dev = _dev()
    K, E = make_calibration(cfg, seed=4)
    K, E = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
    D = cfg.depth_bins
    h1 = torch.from_numpy(make_head(cfg, seed=4)).to(dev)
    h2 = h1.clone()
    h2[:, D:] = torch.from_numpy(make_head(cfg, seed=5)).to(dev)[:, D:]
    h3 = h1.clone()
    h3[:, D:] = 0.5 * h1[:, D:] + h2[:, D:]
    lift = LiftSplat.from_config(cfg).to(dev)
    b1, b2, b3 = lift(h1, K, E), lift(h2, K, E), lift(h3, K, E)
    assert O.normwise_error((0.5 * b1 + b2).cpu(), b3.cpu()) < 1e-5
    # mass conservation: sum over the grid == sum over kept points of prob * ctx  (softmax sums to 1 per pixel)
    _, valid, _ = lift.point_indices(K, E)
    prob = h1[:, :D].softmax(1)                                             # (B*n, D, h, w)
    w = (prob * valid.view(cfg.frames * cfg.n_cameras, D, *cfg.feat_hw)).sum(1, keepdim=True)
    expect = (w * h1[:, D:]).view(cfg.frames, cfg.n_cameras, cfg.out_channels, -1).sum((1, 3))
    got = b1.sum((2, 3))
    assert torch.allclose(got, expect, rtol=1e-4, atol=1e-2)


def test_ragged_width_and_empty_batch():
    """w not a multiple of the 4-column tile edge is handled by zero-filled TMA columns; B' = 0 returns an empty BEV."""
    cfg = LiftConfig("ragged", n_cameras=2, final_dim=(64, 160), x_bound=(-50.0, 50.0, 1.0), y_bound=(-50.0, 50.0, 1.0),
                     frames=1)       # w = 20 = 5 tiles
    assert cfg.feat_hw == (8, 20)
    dev = _dev()
    K, E = make_calibration(cfg, seed=6)
    head = torch.from_numpy(make_head(cfg, seed=6))
    lift = LiftSplat.from_config(cfg).to(dev)
    got = lift(head.to(dev), torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)).cpu()
    exact = O.LiftOracle.from_config(cfg).lift_exact(head, torch.from_numpy(K), torch.from_numpy(E))
    assert O.normwise_error(got, exact) < TOL
    empty = lift(head[:0].to(dev), torch.from_numpy(K[:0]).to(dev), torch.from_numpy(E[:0]).to(dev))
    assert tuple(empty.shape) == (0, cfg.out_channels, *cfg.bev_hw)


def test_graph_capture_and_host_pipeline_match_eager():
    """LiftSplat.capture() (CUDA-graph replay) and LiftSplat.lift_from_host() (pinned host buffers, chunked 3-stream
    pipeline) return what the eager call returns."""
    cfg = LiftConfig(**{**CONFIGS["cfg2_static_lss"].__dict__, "frames": 5})
    dev = _dev()
    K, E = make_calibration(cfg, seed=21)
    head = torch.from_numpy(make_head(cfg, seed=21))
    Kd, Ed, hd = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev), head.to(dev)
    lift = LiftSplat.from_config(cfg).to(dev)
    with torch.no_grad():
        eager = lift(hd, Kd, Ed).clone()
    g = lift.capture(hd, Kd, Ed)
    for _ in range(3):
        replay = g()
    torch.cuda.synchronize()
    assert O.normwise_error(replay.cpu(), eager.cpu()) < 1e-6
    out = lift.lift_from_host(head.pin_memory(), torch.from_numpy(K).pin_memory(), torch.from_numpy(E).pin_memory(),
                              device=dev, chunk_frames=2)
    assert out.is_pinned() and tuple(out.shape) == tuple(eager.shape)
    assert O.normwise_error(out, eager.cpu()) < 1e-6
    # frames are independent: any chunking gives the same result
    out1 = lift.lift_from_host(head.pin_memory(), torch.from_numpy(K).pin_memory(), torch.from_numpy(E).pin_memory(),
                               device=dev, chunk_frames=5)
    assert O.normwise_error(out1, out) < 1e-6


def test_frame_groups_match_frame_by_frame_calls():
    """A batch large enough to be cut into frame groups (tile kernel -> layout pass chains on forked streams,
    lift_fwd.cu:lift_forward_groups) returns, frame for frame, what single-frame calls return, leaves the scratch all-zero,
    and reports its launches through fiery_lift_forward_launches."""
    from fiery_b200 import _lib
    from fiery_b200.geometry import _stream_ptr
    cfg = LiftConfig(**{**CONFIGS["cfg2_static_lss"].__dict__, "frames": 9})
    dev = _dev()
    K, E = make_calibration(cfg, seed=31)
    Kd, Ed = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
    hd = torch.from_numpy(make_head(cfg, seed=31)).to(dev)
    lift = LiftSplat.from_config(cfg).to(dev)
    lib = _lib.load()
    c = lift._constants(dev)
    desc = lift._desc(c, cfg.frames, cfg.n_cameras, torch.float32, _lib.CALIB_RAW, _lib.BEV_NCHW)
    n_launch = int(lib.fiery_lift_forward_launches(desc))
    assert n_launch >= 4 and n_launch % 2 == 0          # more than one (tile kernel, layout pass) chain
    scratch = torch.zeros(int(lib.fiery_lift_scratch_bytes(desc)) // 4, dtype=torch.float32, device=dev)
    X, Y = cfg.bev_hw
    out = torch.full((cfg.frames, cfg.out_channels, X, Y), float("nan"), dtype=torch.float32, device=dev)
    for _ in range(2):                                   # second call: the scratch left by the first must be clean
        _lib.check(lib.fiery_lift_forward(desc, hd.data_ptr(), Kd.data_ptr(), Ed.data_ptr(), c["u"].data_ptr(), c["v"].data_ptr(),
                                          c["d"].data_ptr(), out.data_ptr(), scratch.data_ptr(), None, _stream_ptr(dev)), "fwd")
    torch.cuda.synchronize()
    assert bool((scratch == 0).all())
    n = cfg.n_cameras
    with torch.no_grad():
        for f in range(cfg.frames):
            one = lift(hd[f * n:(f + 1) * n], Kd[f:f + 1], Ed[f:f + 1])
            assert O.normwise_error(out[f:f + 1].cpu(), one.cpu()) < 1e-6, f"frame {f}"
    d1 = lift._desc(c, 1, cfg.n_cameras, torch.float32, _lib.CALIB_RAW, _lib.BEV_NCHW)
    assert int(lib.fiery_lift_forward_launches(d1)) == 2
    d1.bev_layout = _lib.BEV_NHWC
    assert int(lib.fiery_lift_forward_launches(d1)) == 1


def test_row_order_of_the_frustum_is_not_assumed():
    """The kernels pool along image columns but evaluate the geometry of every row: nothing may rely on the frustum's row
    coordinates being sorted (fiery.py:122 makes them a linspace).  A frustum with permuted rows must give the lift of
    exactly that frustum."""
    cfg = LiftConfig(**{**CONFIGS["cfg2_static_lss"].__dict__, "frames": 2})
    dev = _dev()
    K, E = make_calibration(cfg, seed=17)
    head = torch.from_numpy(make_head(cfg, seed=17))
    lift = LiftSplat.from_config(cfg).to(dev)
    oracle = O.LiftOracle.from_config(cfg)
    h = oracle.frustum.shape[1]
    perm = torch.from_numpy(np.random.default_rng(3).permutation(h))
    assert not bool((perm[1:] > perm[:-1]).all())
    oracle.frustum = oracle.frustum[:, perm].contiguous()
    lift.frustum.data = lift.frustum.data[:, perm.to(dev)].contiguous()
    lift._consts = None
    with torch.no_grad():
        got = lift(head.to(dev), torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)).cpu()
    want = oracle.lift_exact(head, torch.from_numpy(K), torch.from_numpy(E))
    assert O.normwise_error(got, want) < TOL
    assert O.max_abs_scaled_error(got, want) < 1e-4


def test_reference_call_site_signature_and_amp_head():
    """fiery_b200.lift.calculate_birds_eye_view_features has the signature and return shape of
    Fiery.calculate_birds_eye_view_features (fiery/models/fiery.py:275-286): x (b,s,n,3,H,W) -> (b,s,C,X,Y).  The stand-in
    model carries the attributes the reference module has (encoder.get_features / depth_layer / use_depth_distribution,
    frustum, bev_*), with a tiny conv as backbone; fp16 head tensors (AMP, baseline.yml PRECISION 16) are accepted."""
    import types
    from fiery_b200.lift import calculate_birds_eye_view_features
    cfg = LiftConfig(**{**CONFIGS["cfg1_tiny"].__dict__, "frames": 2})
    dev = _dev()
    torch.manual_seed(0)
    H, W = cfg.final_dim

    class Enc(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.use_depth_distribution = True
            self.feat = torch.nn.Conv2d(3, 16, 8, stride=8)
            self.depth_layer = torch.nn.Conv2d(16, cfg.head_channels, 1)

        def get_features(self, x):
            return self.feat(x)

    proto = LiftSplat.from_config(cfg)
    model = types.SimpleNamespace(encoder=Enc().to(dev), frustum=proto.frustum, bev_resolution=proto.bev_resolution,
                                  bev_start_position=proto.bev_start_position, bev_dimension=proto.bev_dimension,
                                  encoder_out_channels=cfg.out_channels)
    b, s, n = 1, 2, cfg.n_cameras
    x = torch.randn(b, s, n, 3, H, W, device=dev)
    K, E = make_calibration(cfg, seed=8)
    K = torch.from_numpy(K).view(b, s, n, 3, 3).to(dev)
    E = torch.from_numpy(E).view(b, s, n, 4, 4).to(dev)
    out = calculate_birds_eye_view_features(model, x, K, E)
    assert tuple(out.shape) == (b, s, cfg.out_channels, *cfg.bev_hw)
    with torch.no_grad():
        head = model.encoder.depth_layer(model.encoder.get_features(x.view(b * s * n, 3, H, W)))
    exact = O.LiftOracle.from_config(cfg).lift_exact(head.cpu(), K.view(b * s, n, 3, 3).cpu(), E.view(b * s, n, 4, 4).cpu())
    assert O.normwise_error(out.detach().view(b * s, *out.shape[2:]).cpu(), exact) < TOL
    out.sum().backward()                                   # gradients reach the encoder's parameters through the lift
    assert model.encoder.depth_layer.weight.grad is not None and model.encoder.feat.weight.grad.abs().sum() > 0
    # AMP: fp16 head in, fp32 BEV out, fp16 gradient back
    lift = LiftSplat.from_config(cfg).to(dev)
    h16 = head.half().requires_grad_(True)
    bev16 = lift(h16, K.view(b * s, n, 3, 3), E.view(b * s, n, 4, 4))
    assert bev16.dtype == torch.float32
    exact16 = O.LiftOracle.from_config(cfg).lift_exact(h16.detach().float().cpu(), K.view(b * s, n, 3, 3).cpu(),
                                                       E.view(b * s, n, 4, 4).cpu())
    assert O.normwise_error(bev16.detach().cpu(), exact16) < TOL
    bev16.sum().backward()
    assert h16.grad.dtype == torch.float16


@pytest.mark.parametrize("name,frames,use_depth", [("cfg1_tiny", 2, True), ("cfg1_tiny", 1, False), ("cfg2_static_lss", 1, True),
                                                    ("cfg3_baseline", 9, True)])
def test_half_precision_head_read_by_the_tile_kernel(name, frames, use_depth):
    """fp16 head tensor (AMP, baseline.yml PRECISION 16) through fiery_lift_forward with FIERY_DTYPE_F16: the tile kernel fetches
    the fp16 pieces itself and widens them in shared memory.  Must equal the lift of the exactly widened fp32 tensor (same
    arithmetic; only the accumulation order differs) and match the exact pooling of those values."""
    from fiery_b200 import lift as lift_mod
    cfg = LiftConfig(**{**CONFIGS[name].__dict__, "frames": frames, "use_depth_distribution": use_depth})
    dev = _dev()
    K, E = make_calibration(cfg, seed=41)
    Kd, Ed = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
    h16 = torch.from_numpy(make_head(cfg, seed=41)).to(dev).half()
    lift = LiftSplat.from_config(cfg).to(dev)
    old = lift_mod.NATIVE_FP16_FORWARD
    with torch.no_grad():
        widened = lift(h16.float(), Kd, Ed)
        lift_mod.NATIVE_FP16_FORWARD = True
        try:
            native = lift._launch_forward(h16, Kd, Ed)           # DTYPE_F16 through the C ABI
        finally:
            lift_mod.NATIVE_FP16_FORWARD = old
        default = lift._launch_forward(h16, Kd, Ed)              # default: widened on the device first
    assert native.dtype == torch.float32 and default.dtype == torch.float32
    assert O.normwise_error(default.cpu(), widened.cpu()) < 1e-6
    assert O.normwise_error(native.cpu(), widened.cpu()) < 1e-6
    if frames <= 2:
        exact = O.LiftOracle.from_config(cfg).lift_exact(h16.float().cpu(), torch.from_numpy(K), torch.from_numpy(E))
        assert O.normwise_error(native.cpu(), exact) < TOL
    # the autograd path with the switch on: fp16 in, fp32 BEV, fp16 gradient, same values as the widened path
    lift_mod.NATIVE_FP16_FORWARD = True
    try:
        a = h16.clone().requires_grad_(True)
        out = lift(a, Kd, Ed)
        out.sum().backward()
    finally:
        lift_mod.NATIVE_FP16_FORWARD = old
    b = h16.clone().requires_grad_(True)
    lift(b, Kd, Ed).sum().backward()
    assert a.grad.dtype == torch.float16 and torch.equal(a.grad, b.grad)
    assert O.normwise_error(out.detach().cpu(), widened.cpu()) < 1e-6


def test_all_points_masked_and_degenerate_calibration():
    """Frustum entirely outside the grid -> BEV exactly zero (fiery.py:240-249 drops every point); a non-finite calibration
    masks all points as well (long(NaN) is negative in the reference) instead of corrupting memory."""
    cfg = CONFIGS["cfg1_tiny"]
    dev = _dev()
    K, E = make_calibration(cfg, seed=12)
    head = torch.from_numpy(make_head(cfg, seed=12)).to(dev)
    lift = LiftSplat.from_config(cfg).to(dev)
    far = E.copy()
    far[..., 0, 3] += 1.0e4                                   # rig 10 km ahead of the grid
    bev = lift(head, torch.from_numpy(K).to(dev), torch.from_numpy(far).to(dev))
    assert float(bev.abs().max()) == 0.0
    idx, valid, pillar = lift.point_indices(torch.from_numpy(K).to(dev), torch.from_numpy(far).to(dev))
    assert not bool(valid.any()) and bool((pillar == -1).all())
    oracle = O.LiftOracle.from_config(cfg)
    comb, _ = lift.compose_calibration(torch.from_numpy(K).to(dev), torch.from_numpy(far).to(dev))
    idx_o, keep_o = oracle.point_indices(torch.from_numpy(K), torch.from_numpy(far), combined=comb.cpu())
    assert torch.equal(idx.cpu(), idx_o) and not bool(keep_o.any())
    bad = K.copy()
    bad[0, 0, 0, 0] = float("nan")
    bev = lift(head, torch.from_numpy(bad).to(dev), torch.from_numpy(E).to(dev))
    torch.cuda.synchronize()
    assert float(bev.abs().max()) == 0.0 and bool(torch.isfinite(bev).all())
    # the scratch is still clean afterwards: a normal call gives the normal answer
    good = lift(head, torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)).cpu()
    exact = oracle.lift_exact(head.cpu(), torch.from_numpy(K), torch.from_numpy(E))
    assert O.normwise_error(good, exact) < TOL


def test_lift_is_a_dispatcher_operator():
    """torch.ops.fiery_b200.lift_splat (torch.library.custom_op over the C ABI): autograd formula registered on the operator, fake
    implementation for tracing (torch.compile, fullgraph), autocast rule = fp32 like the reference's softmax / outer product under
    AMP (fiery/models/encoder.py:99-100).  The same for the warped lift (LiftSplat.forward_warped): the operator with the warp's
    theta / copy_mask."""
    from fiery_b200 import ops
    from fiery_b200.synthetic import make_egomotion
    from fiery_b200.warp import _device_theta
    from oracle import warp_oracle as W
    cfg = LiftConfig(**{**CONFIGS["cfg1_tiny"].__dict__, "frames": 2})
    dev = _dev()
    K, E = make_calibration(cfg, seed=3)
    Kd, Ed = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
    head = torch.from_numpy(make_head(cfg, seed=3)).to(dev)
    flow = torch.from_numpy(make_egomotion(1, 2, seed=3))                # one sequence of the two frames
    ext = (float(cfg.x_bound[1]), float(cfg.y_bound[1]))
    warp = _device_theta(flow.to(dev), ext, cumulative=True)
    lift = LiftSplat.from_config(cfg).to(dev)
    handle = ops.register_module(lift, dev)
    oracle = O.LiftOracle.from_config(cfg)

    def warped_exact(h):
        exact = oracle.lift_exact(h, torch.from_numpy(K), torch.from_numpy(E)).float().unflatten(0, (1, 2))
        return W.cumulative_warp_features(exact.clone(), flow, mode="bilinear", spatial_extent=ext).flatten(0, 1)

    for name, extra, module_call, exact_of in (
            ("plain", (), lambda x: lift(x, Kd, Ed),
             lambda h: oracle.lift_exact(h, torch.from_numpy(K), torch.from_numpy(E))),
            ("warped", warp, lambda x: lift.forward_warped(x, Kd, Ed, flow.to(dev), ext).flatten(0, 1), warped_exact)):
        h = head.clone().requires_grad_(True)
        bev, plan = torch.ops.fiery_b200.lift_splat(h, Kd, Ed, None, handle, True, *extra)
        assert plan.numel() > 0 and bev.grad_fn is not None and not plan.requires_grad, name
        bev.sum().backward()
        h2 = head.clone().requires_grad_(True)
        module_call(h2).sum().backward()                            # the module goes through the same operator
        assert torch.equal(h.grad, h2.grad), name
        assert O.normwise_error(bev.detach().cpu(), exact_of(head.cpu())) < TOL, name
        # autocast: an fp16 head inside an autocast region is lifted in fp32; the gradient comes back in fp16
        h16 = head.half().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.float16):
            out = module_call(h16)
        assert out.dtype == torch.float32, name
        out.sum().backward()
        assert h16.grad.dtype == torch.float16, name
        assert O.normwise_error(out.detach().cpu(), exact_of(h16.detach().float().cpu())) < TOL, name
        # traceable: dynamo captures the call as ONE operator node (fake implementation gives shapes / dtypes)
        fn = torch.compile(lambda x: torch.ops.fiery_b200.lift_splat(x, Kd, Ed, None, handle, False, *extra)[0] * 2.0, backend="eager",
                           fullgraph=True)
        with torch.no_grad():
            assert O.normwise_error((fn(head) / 2.0).cpu(), bev.detach().cpu()) < 1e-6, name
