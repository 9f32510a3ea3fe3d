"""GPU: the warped lift (LiftSplat.forward_warped) across the envelope's shapes, forward and backward, against fp64.

The forward (fiery_lift_forward_warped) samples every past frame under its map straight from the lift's accumulator and passes the
present frame through; the backward runs the warp's gather adjoint and then the lift's backward inside one operator.  The oracle is
built per frame from the kernel's own fp32 theta (fiery_warp_theta): the forward is oracle.lift_exact sampled by fp64 grid_sample
(tests/test_warp_envelope_gpu._ref64), copy frames passed through; the gradient is the fp64 autograd gradient of the lift
(tests/test_lift_backward_gpu._oracle_grad) at the fp64 adjoint of the upstream gradient (_ref64_backward).

Bars: the present frame keeps the envelope's bars.  A sampled frame carries one more fp32 stage, the sample position, whose error
tests/test_warp_envelope_gpu._coord_error bounds by (dx, dy) pixels; the warp envelope derives from it a bar on the sampled values of
max|x| (2 (dx + dy) + 8u) and on the adjoint of K max|g| (dx + dy + (K + 4) u), K the adjoint window (16 square, 30 rectangular maps).
Normwise and max-abs-scaled errors keep the 1e-4 bar.  Element-wise, the forward allows 1e-4 relative plus the sampled-value bound;
the gradient allows 1e-4 relative plus the adjoint bound times what the lift's backward can amplify it by at that head element: 1
for a context channel (the depth probabilities of a pixel sum to at most 1), 2 sum_c |context_c| for a depth logit."""
import pytest
import torch

from fiery_b200 import lift as lift_mod
from fiery_b200.lift import LiftSplat
from fiery_b200.synthetic import CONFIGS, make_egomotion
from fiery_b200.warp import _device_theta
from oracle import lift_oracle as O
from tests.test_lift_backward_gpu import _oracle_grad
from tests.test_lift_envelope_gpu import _ORACLE, SHAPES, TOL, _assert_bev, _assert_scratch_clean, _exact, _frames, _inputs
from tests.test_warp_envelope_gpu import U, _coord_error, _ref64, _ref64_backward

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TAG = "warp_envelope"
# one depth bin, one image row, one column tile, 31 rows at D = 48, and the 51 x 49 grid (X*Y % 4 != 0)
SUBSET = ["D1-h8-w16-n1", "D41-h1-w60-n6-101x99", "D45-h3-w4-n5", "D48-h31-w36-n6", "D7-h5-w12-n3-51x49"]
CASES = [(name, b, s) for name in SUBSET for b, s in ((1, 2), (2, 3))]


@pytest.fixture(scope="module", autouse=True)
def _oracle_cache():
    yield
    for k in [k for k in _ORACLE if k[0] == TAG]:
        del _ORACLE[k]


def _make(name, b, s, seed):
    base = CONFIGS[name] if name in CONFIGS else SHAPES[name]
    cfg = _frames(base, b * s)
    head, K, E, gout = _inputs(cfg, seed)
    flow = torch.from_numpy(make_egomotion(b, s, seed=seed))
    ext = (float(cfg.x_bound[1]), float(cfg.y_bound[1]))
    theta, copy = _device_theta(flow.to(DEV), ext, cumulative=True)
    copy = copy.bool().cpu()
    assert int(copy.sum()) == b
    X, Y = cfg.bev_hw
    dx, dy = _coord_error(theta, X, Y)
    return dict(key=(TAG, name, b, s), cfg=cfg, b=b, s=s, head=head, K=K, E=E, gout=gout, flow=flow, ext=ext, theta=theta,
                copy=copy, dxy=(dx + dy).cpu(), window=16 if X == Y else 30, hd=head.to(DEV), Kd=K.to(DEV), Ed=E.to(DEV), fd=flow.to(DEV),
                gd=gout.to(DEV))


@pytest.fixture(scope="module", params=CASES, ids=[f"{n}-{b}x{s}" for n, b, s in CASES])
def case(request):
    name, b, s = request.param
    return _make(name, b, s, seed=300 + CASES.index(request.param))


@pytest.fixture(scope="module")
def baseline():
    """cfg3_baseline, b = 2, s = 4: 8 frames in 4 frame groups on 2 scratch lanes."""
    return _make("cfg3_baseline", 2, 4, seed=390)


def _want_bev(c, head=None, tag=""):
    """(the exact lift, the expected warped BEV) (B', C, X, Y) fp64: every sampled frame through fp64 grid_sample on the kernel's
    theta, the copy frames as they are."""
    exact = _exact(c["key"] + ("lift", tag), c["cfg"], c["head"] if head is None else head, c["K"], c["E"])
    key = c["key"] + ("bev", tag)
    if key not in _ORACLE:
        out = exact.clone()
        for f in (~c["copy"]).nonzero().flatten().tolist():
            out[f] = _ref64(exact[f:f + 1].to(DEV), c["theta"][f:f + 1], 0)[0].cpu()
        _ORACLE[key] = out
    return exact, _ORACLE[key]


def _want_grad(c, gout, tag):
    """fp64 gradient of <warped lift(head), gout> w.r.t. the head, one frame at a time."""
    key = c["key"] + ("grad", tag)
    if key not in _ORACLE:
        cfg, n = c["cfg"], c["cfg"].n_cameras
        parts = []
        for f in range(cfg.frames):
            g = gout[f:f + 1].double()
            if not c["copy"][f]:
                g = _ref64_backward(g.to(DEV), c["theta"][f:f + 1], 0).cpu()
            parts.append(_oracle_grad(cfg, c["head"][f * n:(f + 1) * n], c["K"][f:f + 1], c["E"][f:f + 1], g, exact=True))
        _ORACLE[key] = torch.cat(parts)
    return _ORACLE[key]


def _assert_warped_bev(got, c, oracle, what):
    lifted, want = oracle
    got = got.detach().cpu().flatten(0, 1)
    assert got.shape == want.shape and got.dtype == torch.float32, what
    assert O.normwise_error(got, want) < TOL, (what, O.normwise_error(got, want))
    assert O.max_abs_scaled_error(got, want) < TOL, (what, O.max_abs_scaled_error(got, want))
    for f in range(want.shape[0]):
        if c["copy"][f]:
            _assert_bev(got[f:f + 1], want[f:f + 1], (what, f))
            continue
        xmax = float(lifted[f].abs().max())
        bar = TOL * want[f].abs() + xmax * (2.0 * float(c["dxy"][f]) + 8.0 * U)
        err = (got[f].double() - want[f]).abs()
        assert bool((err <= bar).all()), (what, f, float((err - bar).max()))


def _assert_warped_grad(got, c, want, gout, what):
    got = got.detach().cpu()
    assert got.shape == want.shape, what
    assert O.normwise_error(got, want) < TOL, (what, O.normwise_error(got, want))
    assert O.max_abs_scaled_error(got, want) < TOL, (what, O.max_abs_scaled_error(got, want))
    cfg, n = c["cfg"], c["cfg"].n_cameras
    D = cfg.depth_bins
    K = c["window"]
    gmax = gout.flatten(1).abs().max(1).values.double().cpu()
    adj = torch.where(c["copy"], torch.zeros_like(gmax), K * gmax * (c["dxy"] + (K + 4) * U))       # per frame
    amp = torch.ones_like(c["head"], dtype=torch.float64)
    amp[:, :D] = 2.0 * c["head"][:, D:].double().abs().sum(1, keepdim=True)
    bar = TOL * want.abs() + amp * adj.repeat_interleave(n).view(-1, 1, 1, 1)
    big = want.abs() > 1e-2 * want.abs().max()
    err = (got.double() - want).abs()
    assert bool((err <= bar)[big].all()), (what, float((err - bar)[big].max()))


# ==== forward ====================================================================================================================
@pytest.mark.parametrize("plan", [False, True], ids=["geometry", "plan"])
@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
def test_warped_forward_matches_fp64(case, layout, plan):
    c = case
    cfg = c["cfg"]
    lift = LiftSplat.from_config(cfg, output_layout=layout).to(DEV)
    p = lift.plan(c["Kd"], c["Ed"]) if plan else None
    with torch.no_grad():
        for _ in range(2):                                             # the second call finds the scratch the first one left
            out = lift.forward_warped(c["hd"], c["Kd"], c["Ed"], c["fd"], c["ext"], plan=p)
    assert tuple(out.shape) == (c["b"], c["s"], cfg.out_channels, *cfg.bev_hw) and out.is_contiguous()
    _assert_warped_bev(out, c, _want_bev(c), (layout, plan, False))
    _assert_scratch_clean()


def test_warped_forward_over_four_frame_groups(baseline):
    with torch.no_grad():
        lift = LiftSplat.from_config(baseline["cfg"]).to(DEV)
        out = lift.forward_warped(baseline["hd"], baseline["Kd"], baseline["Ed"], baseline["fd"], baseline["ext"])
    _assert_warped_bev(out, baseline, _want_bev(baseline), ("cfg3", False))
    _assert_scratch_clean()


# ==== backward ===================================================================================================================
def _upstream(c, grad):
    """(upstream gradient as the kernel gets it, its values as a dense tensor)."""
    if grad == "stride0":
        ones = torch.ones(1, device=DEV).expand(c["cfg"].frames, c["cfg"].out_channels, *c["cfg"].bev_hw)
        return ones, ones.contiguous()
    g = c["gd"] if grad == "nchw" else c["gd"].permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    return g, c["gd"]


def _backward(lift, c, grad, plan, head=None):
    h = (c["hd"] if head is None else head).clone().requires_grad_(True)
    out = lift.forward_warped(h, c["Kd"], c["Ed"], c["fd"], c["ext"], plan=plan)
    if grad == "stride0":
        out.sum().backward()                                           # an expanded (stride-0) upstream gradient
    else:
        out.backward(_upstream(c, grad)[0].unflatten(0, (c["b"], c["s"])))
    return h.grad


@pytest.mark.parametrize("grad", ["nchw", "channels_last", "stride0"])
@pytest.mark.parametrize("plan", ["autograd", "caller"])
def test_warped_backward_matches_fp64(case, plan, grad):
    c = case
    lift = LiftSplat.from_config(c["cfg"]).to(DEV)
    p = lift.plan(c["Kd"], c["Ed"]) if plan == "caller" else None
    dense = _upstream(c, grad)[1]
    want = _want_grad(c, dense.cpu(), "ones" if grad == "stride0" else "g")
    _assert_warped_grad(_backward(lift, c, grad, p), c, want, dense, (plan, grad))


def test_warped_backward_of_a_channels_last_module(case):
    """The warped output is NCHW whatever the module's layout; so is the gradient the backward re-lays."""
    c = case
    lift = LiftSplat.from_config(c["cfg"], output_layout="channels_last").to(DEV)
    with torch.no_grad():
        assert lift.forward_warped(c["hd"], c["Kd"], c["Ed"], c["fd"], c["ext"]).is_contiguous()
    _assert_warped_grad(_backward(lift, c, "nchw", None), c, _want_grad(c, c["gout"], "g"), c["gd"], "channels_last module")


def test_warped_backward_over_four_frame_groups(baseline):
    lift = LiftSplat.from_config(baseline["cfg"]).to(DEV)
    _assert_warped_grad(_backward(lift, baseline, "nchw", None), baseline, _want_grad(baseline, baseline["gout"], "g"),
                        baseline["gd"], "cfg3")


@pytest.mark.parametrize("how", ["autocast", "native"])
def test_warped_fp16_head(case, how):
    """An fp16 head: the forward against fp64 on the widened values; the gradient comes back in fp16 and equals the widened head's
    gradient rounded to fp16, bit for bit (the backward reads the same fp32 values under the same plan)."""
    c = case
    h16 = c["hd"].half()
    lift = LiftSplat.from_config(c["cfg"]).to(DEV)
    old = lift_mod.NATIVE_FP16_FORWARD
    lift_mod.NATIVE_FP16_FORWARD = how == "native"
    try:
        h = h16.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.float16, enabled=how == "autocast"):
            out = lift.forward_warped(h, c["Kd"], c["Ed"], c["fd"], c["ext"])
        assert out.dtype == torch.float32
        out.backward(c["gd"].unflatten(0, (c["b"], c["s"])))
    finally:
        lift_mod.NATIVE_FP16_FORWARD = old
    _assert_warped_bev(out, c, _want_bev(c, h16.float().cpu(), "f16"), (how, True))
    assert h.grad.dtype == torch.float16
    wide = _backward(lift, c, "nchw", None, head=h16.float())
    assert torch.equal(h.grad, wide.half())
