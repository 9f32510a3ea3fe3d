"""GPU: the deterministic forward lift (fiery_lift_forward_deterministic, selected by torch.use_deterministic_algorithms(True)).

Every pillar is the fp32 sum of its runs' partial sums, added in ascending (tile, run) order of its own frame, so a frame's BEV must
be bit-identical across calls, workspace contents, batch companions, pass splits, plans, layouts, graph capture, host pipelines and
streams -- and still meet the fp64 oracle's bars of the default path.  "Bit-equal" is torch.equal on the int32 views."""
import contextlib

import pytest
import torch

from fiery_b200 import _lib, ops
from fiery_b200.bev_conv import FirstConv
from fiery_b200.depth_layer import DepthLayer
from fiery_b200.geometry import _stream_ptr
from fiery_b200.lift import LiftSplat
from fiery_b200 import warp as warp_mod
from fiery_b200.synthetic import CONFIGS, LiftConfig, make_egomotion
from oracle import lift_oracle as O
from oracle import warp_oracle as W
from tests.test_lift_envelope_gpu import SHAPES, TOL, _assert_bev, _assert_grad, _exact, _exact_grad, _inputs

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REF = CONFIGS["cfg2_static_lss_b8"]


@contextlib.contextmanager
def deterministic(on=True):
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)


@contextlib.contextmanager
def max_pass_frames(n):
    lib = _lib.load()
    lib.fiery_lift_set_max_chunk_frames(n)
    try:
        yield
    finally:
        lib.fiery_lift_set_max_chunk_frames(0)


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def assert_bit_equal(a, b, what=None):
    assert a.shape == b.shape, what
    assert torch.equal(bits(a), bits(b)), (what, float((a - b).abs().max()))


def det_call(lift, head, K, E, layout="contiguous", plan=None, warp=None, fill=float("nan"), calib=None):
    """One fiery_lift_forward_deterministic call through the C ABI with a workspace filled with `fill` (NaN: its contents must not
    matter).  calib = (mode, a, b) overrides the module's calibration."""
    lib = _lib.load()
    nhwc = layout == "channels_last" and warp is None
    desc, geo = lift._abi_args(DEV, K, E, head.dtype, _lib.BEV_NHWC if nhwc else _lib.BEV_NCHW)
    if calib is not None:
        desc.calib_mode = calib[0]
        geo = (calib[1], calib[2]) + tuple(geo[2:])
    c = lift._constants(DEV)
    X, Y, _ = c["dim"]
    B, C = K.shape[0], lift.encoder_out_channels
    out = torch.full((B, X, Y, C) if nhwc else (B, C, X, Y), float("nan"), device=DEV)
    ws = torch.full((max(1, int(lib.fiery_lift_deterministic_workspace_bytes(desc))) // 4 + 1,), fill, device=DEV)
    _lib.check(lib.fiery_lift_forward_deterministic(desc, head.data_ptr(), *(t.data_ptr() for t in geo), out.data_ptr(), ws.data_ptr(),
                                                    plan.data_ptr() if plan is not None else 0,
                                                    warp[0].data_ptr() if warp is not None else 0,
                                                    warp[1].data_ptr() if warp is not None else 0, _stream_ptr(DEV)),
               "fiery_lift_forward_deterministic")
    return out.permute(0, 3, 1, 2) if nhwc else out


def _case(cfg, seed):
    head, K, E, g = _inputs(cfg, seed)
    return dict(cfg=cfg, head=head, K=K, E=E, g=g, hd=head.to(DEV), Kd=K.to(DEV), Ed=E.to(DEV), gd=g.to(DEV))


CASES = {**SHAPES, "cfg2_static_lss_b8": REF}


@pytest.fixture(scope="module", params=list(CASES), ids=list(CASES))
def case(request):
    c = _case(CASES[request.param], seed=7 + list(CASES).index(request.param))
    c["name"] = request.param
    return c


# ---- 1 + 2. parity with the fp64 oracle, and reproducibility ------------------------------------------------------------------
@pytest.mark.parametrize("head_dtype", ["f32", "f16"])
def test_parity_and_reproducibility(case, head_dtype):
    """NCHW and NHWC, internal and caller plan, fp32 and fp16 heads: frame by frame within the envelope bars of the default path;
    three calls with a NaN-filled workspace and another module's call in between are bit-equal, and so are all the variants."""
    cfg = case["cfg"]
    hd = case["hd"] if head_dtype == "f32" else case["hd"].half()
    m = cfg.frames if head_dtype == "f32" else min(cfg.frames, 2)          # the fp16 head: the oracle of two frames is enough
    n = cfg.n_cameras
    exact = _exact((case["name"], "bev" if head_dtype == "f32" else "f16"), LiftConfig(**{**cfg.__dict__, "frames": m}),
                   hd[:m * n].float().cpu(), case["K"][:m], case["E"][:m])
    lift = LiftSplat.from_config(cfg).to(DEV)
    other = LiftSplat.from_config(CASES["D7-h5-w12-n3-51x49"]).to(DEV)
    oc = _case(CASES["D7-h5-w12-n3-51x49"], seed=3)
    plan = lift.plan(case["Kd"], case["Ed"])
    first = None
    for layout in ("contiguous", "channels_last"):
        for p in (None, plan):
            runs = []
            for _ in range(3):
                runs.append(det_call(lift, hd, case["Kd"], case["Ed"], layout, plan=p))
                det_call(other, oc["hd"], oc["Kd"], oc["Ed"], layout)
            for r in runs[1:]:
                assert_bit_equal(r, runs[0], (layout, p is None))
            first = runs[0] if first is None else first
            assert_bit_equal(runs[0], first, (layout, p is None))      # NCHW == NHWC, caller plan == internal plan
    for f in range(m):
        _assert_bev(first[f:f + 1], exact[f:f + 1], (case["name"], f))


def test_operator_follows_the_flag(case):
    """LiftSplat.forward under the flag equals the C-ABI call bit for bit, and the uniform-depth / fp16 paths come through too."""
    lift = LiftSplat.from_config(case["cfg"], output_layout="channels_last").to(DEV)
    with deterministic(), torch.no_grad():
        a = lift(case["hd"], case["Kd"], case["Ed"])
        b = lift(case["hd"].half(), case["Kd"], case["Ed"])              # widened on the device, then the same call
    assert_bit_equal(a, det_call(lift, case["hd"], case["Kd"], case["Ed"], "channels_last"))
    assert_bit_equal(b, det_call(lift, case["hd"].half().float(), case["Kd"], case["Ed"], "channels_last"))
    assert not a.is_contiguous() and a.permute(0, 2, 3, 1).is_contiguous()


# ---- 3. invariance --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    c = _case(REF, seed=7 + list(CASES).index("cfg2_static_lss_b8"))      # the inputs of the parity case: one oracle for both
    c["lift"] = LiftSplat.from_config(REF).to(DEV)
    c["base"] = det_call(c["lift"], c["hd"], c["Kd"], c["Ed"])
    return c


def test_frame_alone_equals_frame_in_batch(ref):
    n = REF.n_cameras
    for f in (0, 5, 7):
        alone = det_call(ref["lift"], ref["hd"][f * n:(f + 1) * n], ref["Kd"][f:f + 1], ref["Ed"][f:f + 1])
        assert_bit_equal(alone[0], ref["base"][f], f)


@pytest.mark.parametrize("frames", [1, 2, 3])
def test_forced_passes_equal_one_pass(ref, frames):
    with max_pass_frames(frames):
        lift = ref["lift"]
        c = lift._constants(DEV)
        desc = lift._desc(c, 8, REF.n_cameras, torch.float32, _lib.CALIB_RAW, _lib.BEV_NCHW)
        forced = int(_lib.load().fiery_lift_deterministic_workspace_bytes(desc))
        assert_bit_equal(det_call(lift, ref["hd"], ref["Kd"], ref["Ed"]), ref["base"], frames)
        assert_bit_equal(det_call(lift, ref["hd"], ref["Kd"], ref["Ed"], "channels_last", plan=lift.plan(ref["Kd"], ref["Ed"])),
                         ref["base"], frames)
    assert forced < int(_lib.load().fiery_lift_deterministic_workspace_bytes(desc))


@pytest.mark.parametrize("static", [False, True], ids=["dynamic", "static"])
@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
def test_graph_replay_equals_eager(ref, static, layout):
    lift = LiftSplat.from_config(REF, output_layout=layout).to(DEV)
    with deterministic():
        g = lift.capture(ref["hd"], ref["Kd"], ref["Ed"], static_calibration=static)
    for _ in range(2):
        assert_bit_equal(g(), ref["base"], (static, layout))             # replays outside the flag: captured at capture time


@pytest.mark.parametrize("chunks", [1, [2, 5, 1], 3], ids=["1", "2-5-1", "3"])
def test_host_pipeline_equals_one_device_call(ref, chunks):
    with deterministic():
        out = ref["lift"].lift_from_host(ref["head"].pin_memory(), ref["K"], ref["E"], device=DEV, chunk_frames=chunks)
    assert_bit_equal(out, ref["base"].cpu(), chunks)


def test_two_modules_on_two_streams(ref):
    a, b = LiftSplat.from_config(REF).to(DEV), LiftSplat.from_config(REF, output_layout="channels_last").to(DEV)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    with deterministic(), torch.no_grad():
        for _ in range(3):
            for m, s in ((a, s1), (b, s2)):
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):
                    outs.append(m(ref["hd"], ref["Kd"], ref["Ed"]))
        torch.cuda.synchronize()
    for o in outs:
        assert_bit_equal(o, ref["base"])


@pytest.mark.parametrize("plan", [False, True], ids=["internal", "caller"])
def test_warped_lift(ref, plan):
    """forward_warped under the flag: the present frames equal the plain deterministic BEV bit for bit; the warped frames meet the
    bars of the warped-lift envelope against the fp64 lift warped by the fp64 warp; three calls are bit-equal."""
    b, s = 2, 4
    lift, cfg = ref["lift"], REF
    flow = torch.from_numpy(make_egomotion(b, s, seed=5))
    ext = (float(cfg.x_bound[1]), float(cfg.y_bound[1]))
    p = lift.plan(ref["Kd"], ref["Ed"]) if plan else None
    with deterministic(), torch.no_grad():
        outs = [lift.forward_warped(ref["hd"], ref["Kd"], ref["Ed"], flow.to(DEV), ext, plan=p) for _ in range(3)]
    for o in outs[1:]:
        assert_bit_equal(o, outs[0])
    theta, copy_mask = warp_mod._device_theta(flow.to(DEV), ext, cumulative=True)
    assert_bit_equal(det_call(lift, ref["hd"], ref["Kd"], ref["Ed"], warp=(theta, copy_mask), plan=p).unflatten(0, (b, s)), outs[0])
    fused = outs[0].cpu()
    for q in range(b):
        assert_bit_equal(fused[q, s - 1], ref["base"][q * s + s - 1].cpu(), q)      # the present frame of each sequence
    exact = _exact(("cfg2_static_lss_b8", "bev"), cfg, ref["head"], ref["K"], ref["E"]).unflatten(0, (b, s))
    want = W.cumulative_warp_features(exact.clone().float(), flow, mode="bilinear", spatial_extent=ext)
    assert float((fused - want).abs().max()) <= TOL * float(want.abs().max())
    assert O.normwise_error(fused, want) < TOL


# ---- 4. adversarial geometry and pass counts ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cfg2_static_lss", "D45-h3-w4-n5"])
def test_every_point_in_one_pillar(name):
    """combined = 0 sends every frustum point of a camera to its translation: one pillar receives every run of the frame (17 280 runs
    at the reference shape: the in-place sort of long lists; a few hundred at the small shape: the shared-memory sort).  Reproducible,
    and equal to the fp64 sum of every point's depth-weighted context."""
    cfg = LiftConfig(**{**(CONFIGS.get(name) or SHAPES[name]).__dict__, "frames": 2})
    c = _case(cfg, seed=13)
    lift = LiftSplat.from_config(cfg).to(DEV)
    B, n = 2, cfg.n_cameras
    comb = torch.zeros(B, n, 3, 3, device=DEV)
    trans = torch.tensor([1.3, -2.7, 0.0], device=DEV).expand(B, n, 3).contiguous()
    calib = (_lib.CALIB_COMPOSED, comb, trans)
    runs = [det_call(lift, c["hd"], c["Kd"], c["Ed"], layout, calib=calib) for layout in ("contiguous", "channels_last", "contiguous")]
    for r in runs[1:]:
        assert_bit_equal(r, runs[0])
    got = runs[0].cpu().flatten(2)                                        # (B, C, X*Y)
    occupied = got.abs().sum(1) > 0
    assert int(occupied.sum()) == B and bool((occupied.sum(1) == 1).all())
    D = cfg.depth_bins
    h = c["head"].double().view(B, n, D + 64, *cfg.feat_hw)
    prob = torch.softmax(h[:, :, :D], dim=2).sum(2, keepdim=True)
    exact = (prob * h[:, :, D:]).sum((1, 3, 4))                          # (B, C)
    for f in range(B):
        col = got[f][:, occupied[f]].squeeze(1).double()
        err = float((col - exact[f]).abs().max() / exact[f].abs().max())
        assert err < TOL, (f, err)


def test_all_points_masked_and_empty_batch():
    cfg = SHAPES["D7-h5-w12-n3-51x49"]
    c = _case(cfg, seed=17)
    lift = LiftSplat.from_config(cfg).to(DEV)
    comb = torch.zeros(cfg.frames, cfg.n_cameras, 3, 3, device=DEV)
    trans = torch.full((cfg.frames, cfg.n_cameras, 3), 1e4, device=DEV)
    for layout in ("contiguous", "channels_last"):
        out = det_call(lift, c["hd"], c["Kd"], c["Ed"], layout, calib=(_lib.CALIB_COMPOSED, comb, trans))
        assert torch.equal(bits(out), torch.zeros_like(bits(out)))       # exact +0.0 everywhere
    with deterministic(), torch.no_grad():
        empty = lift(c["hd"][:0], c["Kd"][:0], c["Ed"][:0])
    assert empty.shape == (0, 64, *cfg.bev_hw)


@pytest.mark.parametrize("name", ["cfg3_baseline", "cfg4_pon"])
def test_batches_of_several_passes(name):
    cfg = CONFIGS[name]
    c = _case(cfg, seed=23)
    lift = LiftSplat.from_config(cfg).to(DEV)
    desc = lift._desc(lift._constants(DEV), cfg.frames, cfg.n_cameras, torch.float32, _lib.CALIB_RAW, _lib.BEV_NCHW)
    tpf = cfg.n_cameras * ((cfg.feat_hw[1] + 3) // 4)
    rows = cfg.frames * tpf * 192 * cfg.feat_hw[0]
    assert int(_lib.load().fiery_lift_deterministic_workspace_bytes(desc)) < rows * 256      # more than one pass
    a = det_call(lift, c["hd"], c["Kd"], c["Ed"])
    assert_bit_equal(det_call(lift, c["hd"], c["Kd"], c["Ed"], "channels_last"), a)
    n = cfg.n_cameras
    last = cfg.frames - 1
    assert_bit_equal(det_call(lift, c["hd"][last * n:], c["Kd"][last:], c["Ed"][last:])[0], a[last])
    for f in (0, last):
        _assert_bev(a[f:f + 1], O.LiftOracle.from_config(cfg).lift_exact(c["head"][f * n:(f + 1) * n], c["K"][f:f + 1],
                                                                          c["E"][f:f + 1]), (name, f))


# ---- 5. dispatch ----------------------------------------------------------------------------------------------------------------
def _kernel_names(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events()}


def test_flag_selects_the_deterministic_kernels(ref):
    lift = ref["lift"]
    with torch.no_grad():
        with deterministic():
            on = _kernel_names(lambda: lift(ref["hd"], ref["Kd"], ref["Ed"]))
        off = _kernel_names(lambda: lift(ref["hd"], ref["Kd"], ref["Ed"]))
    assert any("det_reduce_kernel" in k for k in on), sorted(on)
    assert not any("det_" in k for k in off), sorted(off)


def test_autograd_and_compile_under_the_flag():
    cfg = SHAPES["D47-h2-w36-n6"]
    c = _case(cfg, seed=29)
    exact = _exact(("D47-h2-w36-n6", "bev", 29), cfg, c["head"], c["K"], c["E"])
    gexact = _exact_grad(("D47-h2-w36-n6", "grad", 29), cfg, c["head"], c["K"], c["E"], c["g"])
    lift = LiftSplat.from_config(cfg).to(DEV)
    handle = ops.register_module(lift, DEV)
    fn = torch.compile(lambda x: torch.ops.fiery_b200.lift_splat(x, c["Kd"], c["Ed"], None, handle, True)[0], backend="eager",
                       fullgraph=True)
    outs, grads = [], []
    with deterministic():
        for f in (lambda x: lift(x, c["Kd"], c["Ed"]), fn, fn):
            hd = c["hd"].clone().requires_grad_(True)
            bev = f(hd)
            bev.backward(c["gd"])
            outs.append(bev.detach())
            grads.append(hd.grad)
    for o, g in zip(outs[1:], grads[1:]):
        assert_bit_equal(o, outs[0])
        assert_bit_equal(g, grads[0])
    _assert_bev(outs[0], exact, "autograd")
    _assert_grad(grads[0], gexact, "autograd")


@pytest.mark.parametrize("warped", [False, True], ids=["plain", "warped"])
def test_depth_layer_lift_first_conv_chain(monkeypatch, warped):
    """DepthLayer -> lift -> FirstConv (eval), with the backward through the lift and the depth layer: bit-equal over three runs."""
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")             # torch's condition for deterministic cuBLAS calls
    cfg = LiftConfig(**{**REF.__dict__, "frames": 4})
    torch.manual_seed(0)
    D = cfg.depth_bins
    depth = DepthLayer(D + 64).to(DEV)
    conv = FirstConv(bn=torch.nn.BatchNorm2d(64).eval(), relu=True).to(DEV).eval()
    lift = LiftSplat.from_config(cfg, output_layout="contiguous" if warped else "channels_last").to(DEV)
    feat = torch.randn(cfg.frames * cfg.n_cameras, 128, *cfg.feat_hw, device=DEV)
    c = _case(cfg, seed=31)
    flow = torch.from_numpy(make_egomotion(1, cfg.frames, seed=3)).to(DEV)
    ext = (float(cfg.x_bound[1]), float(cfg.y_bound[1]))
    results = []
    with deterministic():
        for _ in range(3):
            depth.zero_grad()
            f = feat.clone().requires_grad_(True)
            head = depth(f)
            if warped:
                bev = lift.forward_warped(head, c["Kd"], c["Ed"], flow, ext).flatten(0, 1)
            else:
                bev = lift(head, c["Kd"], c["Ed"])
            y = conv(bev.contiguous(memory_format=torch.channels_last))
            (bev * torch.linspace(-1, 1, bev.shape[-1], device=DEV)).sum().backward()
            results.append((y, f.grad, depth.weight.grad.clone()))
    for r in results[1:]:
        for a, b in zip(r, results[0]):
            assert_bit_equal(a, b)
