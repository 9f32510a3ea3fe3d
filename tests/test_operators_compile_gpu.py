"""GPU: the four dispatcher operators of fiery_b200/ops.py (lift_splat, lift_splat_backward, first_conv, first_conv_backward) under the
tracing stack -- FakeTensor, AOTAutograd, inductor -- against eager and fp64.

torch.compile plans every buffer, stride and saved tensor from an operator's fake implementation alone; a fake that disagrees with
the real output stops a compiled step at inductor's size / stride assertion, or, where no assertion is emitted, lets the graph go on
with the wrong layout.  So:
  A. every call of a matrix runs for real and under FakeTensorMode on fake copies of its arguments: each output's dtype, device,
     shape and strides must agree (the check is inductor's own, assert_size_stride: strides of dimensions of size > 1), a plan must
     hold exactly fiery_lift_plan_bytes bytes, and torch.library.opcheck passes with its default tests;
  B. compiled forward + backward (aot_eager and inductor, fullgraph) of the loss sum(out * r): the upstream gradient is exactly r on
     every backend, so under torch.use_deterministic_algorithms the BEV and the head's gradient are bit-identical to eager, and they
     meet the fp64 bars of the lift envelope;
  C. the module and the training step compiled the way users compile them (default settings, graph breaks allowed)."""

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F
import torch.utils._pytree as pytree
from torch._C._dynamo.guards import assert_size_stride
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.testing._internal.optests.generate_tests import DEFAULT_TEST_UTILS

from fiery_b200 import _lib, ops
from fiery_b200.bev_conv import FirstConv
from fiery_b200.lift import LiftSplat, _plan_bytes
from fiery_b200.synthetic import CONFIGS, make_egomotion
from fiery_b200.train import LiftTrainer, synthetic_batch
from fiery_b200.warp import _device_theta
from oracle import lift_oracle as O
from tests.test_lift_deterministic_gpu import assert_bit_equal, deterministic
from tests.test_lift_envelope_gpu import SHAPES, _assert_bev, _assert_grad, _exact, _exact_grad, _frames, _inputs
from tests.test_lift_warp_envelope_gpu import _assert_warped_bev, _assert_warped_grad, _make, _want_bev, _want_grad
from tests.test_tensor_core_envelope_gpu import TRAIN_CFG, TRAIN_GRAD_TOL, _replica_loss_and_grads

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# B' * X * Y is not a multiple of 128 for any B' > 0: the touched maps' rounding shows in the plan's size
NAME = "D7-h5-w12-n3-51x49"
CFG = SHAPES[NAME]
WARP_SEED = 47                  # the warped cases share one set of inputs: the warp envelope's oracle cache is keyed by shape only

@pytest.fixture(autouse=True, scope="module")
def _no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old

@pytest.fixture(autouse=True)
def _fresh_dynamo():
    torch._dynamo.reset()                                   # every case compiles from scratch: the recompile limit is never reached
    yield
    torch._dynamo.reset()

def _nerr(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))

# ==== A. fake against real, and opcheck ==========================================================================================
def _fake_vs_real(op, args):
    """Runs ``op`` for real and under FakeTensorMode; every output must agree in dtype, device, shape and strides."""
    real = pytree.tree_leaves(op(*args))
    mode = FakeTensorMode()
    fargs = pytree.tree_map_only(torch.Tensor, mode.from_tensor, args)
    with mode:
        fake = pytree.tree_leaves(op(*fargs))
    assert len(real) == len(fake)
    for i, (r, f) in enumerate(zip(real, fake)):
        assert (r.dtype, r.device) == (f.dtype, f.device), (i, r.dtype, f.dtype, r.device, f.device)
        assert_size_stride(r, tuple(f.shape), tuple(f.stride()))
    return real

def _plan_want(lift, B, n):
    desc = lift._desc(lift._constants(DEV), B, n, torch.float32, _lib.CALIB_RAW, _lib.BEV_NCHW)
    return int(_lib.load().fiery_lift_plan_bytes(desc))

@pytest.fixture(scope="module")
def frames3():
    head, K, E, g = _inputs(_frames(CFG, 3), seed=41)
    return dict(hd=head.to(DEV), Kd=K.to(DEV), Ed=E.to(DEV), gd=g.to(DEV))

LIFT_CALLS = [(B, how, layout, dt, False) for B in (0, 1, 3) for how in ("none", "make", "caller")
              for layout in ("contiguous", "channels_last") for dt in ("f32", "f16")]
LIFT_CALLS += [(3, how, layout, dt, True) for how in ("none", "make", "caller") for layout in ("contiguous", "channels_last")
               for dt in ("f32", "f16")]

def _lift_args(frames3, B, how, layout, dt, warped, requires_grad=False):
    lift = LiftSplat.from_config(CFG, output_layout=layout).to(DEV)
    n = CFG.n_cameras
    head = frames3["hd"][:B * n]
    head = (head.half() if dt == "f16" else head).clone().requires_grad_(requires_grad)
    K, E = frames3["Kd"][:B], frames3["Ed"][:B]
    plan = lift.plan(K, E) if how == "caller" else None
    theta = copy_mask = None
    if warped:
        flow = torch.from_numpy(make_egomotion(1, B, seed=B)).to(DEV)
        theta, copy_mask = _device_theta(flow, (float(CFG.x_bound[1]), float(CFG.y_bound[1])), cumulative=True)
    return lift, (head, K, E, plan, ops.register_module(lift, DEV), how == "make", theta, copy_mask)

@pytest.mark.parametrize("B,how,layout,dt,warped", LIFT_CALLS, ids=["-".join(map(str, c)) for c in LIFT_CALLS])
def test_lift_splat_fake_matches_real(frames3, B, how, layout, dt, warped):
    lift, args = _lift_args(frames3, B, how, layout, dt, warped)
    with deterministic():
        bev, plan = _fake_vs_real(torch.ops.fiery_b200.lift_splat.default, args)
    assert plan.numel() == (_plan_want(lift, B, CFG.n_cameras) if how == "make" else 0)
    assert plan.numel() == (_plan_bytes(B, CFG.n_cameras, CFG.feat_hw[1], CFG.bev_hw[0] * CFG.bev_hw[1]) if how == "make" else 0)
    assert bev.shape == (B, 64, *CFG.bev_hw)
    if B and layout == "channels_last" and not warped:
        assert bev.permute(0, 2, 3, 1).is_contiguous()
    elif B:
        assert bev.is_contiguous()

@pytest.mark.parametrize("B,how,layout,dt,warped", LIFT_CALLS, ids=["-".join(map(str, c)) for c in LIFT_CALLS])
def test_lift_splat_opcheck(frames3, B, how, layout, dt, warped):
    """opcheck's default tests.  A plan made here is left out of the eager-vs-AOT comparison only: its tile records are written up to
    their run counts (fiery_b200/csrc/lift_plan.cuh), so two plans of one calibration agree on every byte the kernels read and not
    on the rest; the BEV and the gradient that plan yields are compared bit for bit in part B."""
    lift, args = _lift_args(frames3, B, how, layout, dt, warped, requires_grad=True)
    tests = [t for t in DEFAULT_TEST_UTILS if not (how == "make" and B and t == "test_aot_dispatch_dynamic")]
    with deterministic():
        torch.library.opcheck(torch.ops.fiery_b200.lift_splat.default, args, test_utils=tests)

BWD_CALLS = [(grad, head, dt, how) for grad in ("nchw", "channels_last", "expand") for head in ("nchw", "channels_last")
             for dt in ("f32", "f16") for how in ("none", "plan", "warped")]

def _backward_args(frames3, grad, head_layout, dt, how):
    """(module, operator arguments): the caller holds the module, the handle only names it."""
    B = 2
    lift, (head, K, E, plan, handle, _, theta, copy_mask) = _lift_args(frames3, B, "caller" if how == "plan" else "none",
                                                                     "contiguous", dt, how == "warped")
    if how == "none":
        plan = torch.empty(0, dtype=torch.uint8, device=DEV)           # what the forward saves when it made no plan
    if head_layout == "channels_last":
        head = head.contiguous(memory_format=torch.channels_last)
    g = frames3["gd"][:B]
    if grad == "channels_last":
        g = g.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    elif grad == "expand":
        g = g[:1, :, :1, :1].expand(B, -1, *CFG.bev_hw)                 # stride 0: the upstream gradient of a sum
    return lift, (head, K, E, g, plan, handle, theta, copy_mask)

@pytest.mark.parametrize("grad,head,dt,how", BWD_CALLS, ids=["-".join(c) for c in BWD_CALLS])
def test_lift_splat_backward_fake_matches_real(frames3, grad, head, dt, how):
    lift, args = _backward_args(frames3, grad, head, dt, how)
    (out,) = _fake_vs_real(torch.ops.fiery_b200.lift_splat_backward.default, args)
    assert out.is_contiguous() and out.dtype == args[0].dtype and out.shape == args[0].shape
    torch.library.opcheck(torch.ops.fiery_b200.lift_splat_backward.default, args)

CONV_CALLS = [(dt, layout, B, hw) for dt in ("f32", "f16", "bf16") for layout in ("nchw", "channels_last")
              for B, hw in ((2, (33, 65)), (0, (20, 18)))]
DTYPES = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}

def _conv_x(B, hw, dt, layout, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 64, *hw, generator=g).to(DEV, DTYPES[dt])
    return x.contiguous(memory_format=torch.channels_last) if layout == "channels_last" else x

def _conv_w(seed=1):
    return (torch.randn(64, 64, 7, 7, generator=torch.Generator().manual_seed(seed)) * 0.02).to(DEV)

@pytest.mark.parametrize("dt,layout,B,hw", CONV_CALLS, ids=[f"{d}-{lay}-B{b}-{h}x{w}" for d, lay, b, (h, w) in CONV_CALLS])
def test_first_conv_fake_matches_real(dt, layout, B, hw):
    x, w = _conv_x(B, hw, dt, layout), _conv_w()
    (y,) = _fake_vs_real(torch.ops.fiery_b200.first_conv.default, (x, w))
    assert y.shape == (B, 64, (hw[0] + 1) // 2, (hw[1] + 1) // 2) and y.dtype == torch.float32
    assert y.permute(0, 2, 3, 1).is_contiguous()
    torch.library.opcheck(torch.ops.fiery_b200.first_conv.default, (x.requires_grad_(True), w.requires_grad_(True)))

CONV_BWD_CALLS = [(ni, nw, dt, gl) for ni in (False, True) for nw in (False, True) for dt in ("f32", "f16")
                  for gl in ("channels_last", "nchw")]

@pytest.mark.parametrize("need_input,need_weight,dt,grad", CONV_BWD_CALLS,
                         ids=[f"in{int(a)}-w{int(b)}-{d}-{g}" for a, b, d, g in CONV_BWD_CALLS])
def test_first_conv_backward_fake_matches_real(need_input, need_weight, dt, grad):
    """(False, False) included: the two empty outputs must be two tensors (an operator's outputs may not alias each other)."""
    x, w = _conv_x(2, (33, 65), dt, "nchw"), _conv_w()
    gy = _conv_x(2, (17, 33), "f32", grad, seed=2)
    args = (gy, x, w, need_input, need_weight)
    gx, gw = _fake_vs_real(torch.ops.fiery_b200.first_conv_backward.default, args)
    assert gx.numel() == (x.numel() if need_input else 0) and gw.numel() == (w.numel() if need_weight else 0)
    if need_input:
        assert gx.dtype == x.dtype and gx.permute(0, 2, 3, 1).is_contiguous()
    torch.library.opcheck(torch.ops.fiery_b200.first_conv_backward.default, args)

# ==== B. compiled forward + backward against eager and fp64 ======================================================================
BACKENDS = ["aot_eager", "inductor"]

def _run(fn, head):
    """(BEV, head gradient) of ``fn(h) -> (bev, loss)``."""
    h = head.detach().clone().requires_grad_(True)
    bev, loss = fn(h)
    loss.backward()
    return bev.detach(), h.grad

def _eager_and_compiled(fn, head, backend):
    with deterministic():
        want = _run(fn, head)
        got = _run(torch.compile(fn, backend=backend, fullgraph=True), head)
    for a, b, what in zip(got, want, ("bev", "grad")):
        assert a.shape == b.shape and a.dtype == b.dtype, what
        assert_bit_equal(a, b, what)
    return got

@pytest.fixture(scope="module")
def plain():
    head, K, E, g = _inputs(CFG, seed=43)
    return dict(head=head, K=K, E=E, g=g, hd=head.to(DEV), Kd=K.to(DEV), Ed=E.to(DEV), gd=g.to(DEV),
                exact=_exact((NAME, "compile", "bev"), CFG, head, K, E), gexact=_exact_grad((NAME, "compile", "grad"), CFG, head, K, E, g))

LIFT_COMPILE = ["make-contiguous", "make-channels_last", "caller", "fp16-autocast", "channels_last-head"]

@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("case", LIFT_COMPILE)
def test_compiled_lift_training_matches_eager_and_fp64(plain, case, backend):
    layout = "channels_last" if case == "make-channels_last" else "contiguous"
    lift = LiftSplat.from_config(CFG, output_layout=layout).to(DEV)
    handle = ops.register_module(lift, DEV)
    K, E, r = plain["Kd"], plain["Ed"], plain["gd"]
    plan = lift.plan(K, E) if case == "caller" else None
    head = plain["hd"]
    if case == "fp16-autocast":
        head = head.half()
    elif case == "channels_last-head":
        head = head.contiguous(memory_format=torch.channels_last)

    def fn(h):
        with torch.autocast("cuda", dtype=torch.float16, enabled=case == "fp16-autocast"):
            bev = torch.ops.fiery_b200.lift_splat(h, K, E, plan, handle, plan is None)[0]
        return bev, (bev * r).sum()

    bev, grad = _eager_and_compiled(fn, head, backend)
    assert grad.dtype == head.dtype
    if case == "fp16-autocast":                                      # the head is widened exactly: the fp32 lift of the same values
        with deterministic():
            wide_bev, wide_grad = _run(fn, head.float())
        assert_bit_equal(bev, wide_bev)
        assert_bit_equal(grad, wide_grad.half())
        exact = _exact((NAME, "compile", "f16"), CFG, head.float().cpu(), plain["K"], plain["E"])
        _assert_bev(bev, exact, case)
        _assert_grad(wide_grad, _exact_grad((NAME, "compile", "f16grad"), CFG, head.float().cpu(), plain["K"], plain["E"], plain["g"]),
                     case)
        return
    _assert_bev(bev, plain["exact"], case)
    _assert_grad(grad, plain["gexact"], case)

@pytest.mark.parametrize("backend", BACKENDS)
def test_compiled_warped_lift_training_matches_eager_and_fp64(backend):
    c = _make(NAME, 2, 2, seed=WARP_SEED)
    lift = LiftSplat.from_config(c["cfg"]).to(DEV)
    handle = ops.register_module(lift, DEV)
    theta, copy_mask = _device_theta(c["fd"], c["ext"], cumulative=True)

    def fn(h):
        bev = torch.ops.fiery_b200.lift_splat(h, c["Kd"], c["Ed"], None, handle, True, theta, copy_mask)[0]
        return bev, (bev * c["gd"]).sum()

    bev, grad = _eager_and_compiled(fn, c["hd"], backend)
    _assert_warped_bev(bev.unflatten(0, (2, 2)), c, _want_bev(c), backend)
    _assert_warped_grad(grad, c, _want_grad(c, c["gout"], "g"), c["gout"], backend)

@pytest.mark.parametrize("backend", BACKENDS)
def test_dynamic_batch_has_a_symbolic_plan(backend, frames3):
    """One dynamic=True function at B' = 1, 2, 3: the plan the fake returns is sized from the symbolic B', so B' = 3 runs the graph
    compiled for B' = 2 (B' = 1 is specialised by dynamo) and every call is bit-identical to eager."""
    cfg = _frames(CFG, 3)
    lift = LiftSplat.from_config(cfg).to(DEV)
    handle = ops.register_module(lift, DEV)
    n = cfg.n_cameras
    head, K, E, g = (t.cpu() for t in (frames3["hd"], frames3["Kd"], frames3["Ed"], frames3["gd"]))

    def fn(h, K, E, r):
        bev = torch.ops.fiery_b200.lift_splat(h, K, E, None, handle, True)[0]
        return bev, (bev * r).sum()

    compiled = torch.compile(fn, backend=backend, dynamic=True, fullgraph=True)
    exact = _exact((NAME, "compile", "frames3"), cfg, head, K, E)
    gexact = _exact_grad((NAME, "compile", "frames3grad"), cfg, head, K, E, g)
    graphs = []
    for B in (1, 2, 3):
        args = (frames3["Kd"][:B], frames3["Ed"][:B], frames3["gd"][:B])
        with deterministic():
            want = _run(lambda h: fn(h, *args), frames3["hd"][:B * n])
            got = _run(lambda h: compiled(h, *args), frames3["hd"][:B * n])
        graphs.append(torch._dynamo.utils.counters["stats"]["unique_graphs"])
        for a, b in zip(got, want):
            assert_bit_equal(a, b, B)
        _assert_bev(got[0], exact[:B], B)
        _assert_grad(got[1], gexact[:B * n], B)
    assert graphs[2] == graphs[1], graphs                             # no recompilation for B' = 3

def test_compiled_first_conv_training_matches_fp64():
    torch.manual_seed(9)
    m = FirstConv().to(DEV)
    x = torch.randn(2, 64, 101, 99, device=DEV).contiguous(memory_format=torch.channels_last)
    r = torch.randn(2, 64, 51, 50, device=DEV)

    def grads(f):
        xi = x.clone().requires_grad_(True)
        m.weight.grad = None
        y = f(xi)
        (y * r).sum().backward()
        return y.detach(), xi.grad, m.weight.grad.clone()

    eager = grads(m)
    got = grads(torch.compile(m, backend="inductor", fullgraph=True))
    for a, b in zip(got, eager):                                      # the same kernels on the same operands
        assert torch.equal(a, b)
    x64 = x.double().requires_grad_(True)
    w64 = m.weight.detach().double().requires_grad_(True)
    y64 = F.conv2d(x64, w64, stride=2, padding=3)
    (y64 * r.double()).sum().backward()
    assert _nerr(got[0], y64) < 1e-3
    for a, want in ((got[1], x64.grad), (got[2], w64.grad)):
        assert _nerr(a, want) < 1e-3
        assert float((a.double().cpu() - want.cpu()).abs().max()) < 2e-3 * float(want.abs().max())

def test_compiled_lift_first_conv_bn_relu_chain():
    """The lift -> FirstConv -> BN (training statistics) -> relu chain at cfg1_tiny, 2 frames, under inductor: gradients within 2e-3
    of eager.  Eager takes the relu's mask from the compiled run (a reordered BN reduction may flip the sign of a value near 0)."""
    cfg = _frames(CONFIGS["cfg1_tiny"], 2)
    head, K, E, _ = _inputs(cfg, seed=53)
    torch.manual_seed(3)
    lift = LiftSplat.from_config(cfg, output_layout="channels_last").to(DEV)
    conv, bn = FirstConv().to(DEV), nn.BatchNorm2d(64).to(DEV).train()
    handle = ops.register_module(lift, DEV)
    Kd, Ed = K.to(DEV), E.to(DEV)

    def chain(h, mask=None):
        pre = bn(conv(torch.ops.fiery_b200.lift_splat(h, Kd, Ed, None, handle, True)[0]))
        out = torch.relu(pre) if mask is None else pre * mask
        r = torch.linspace(-1, 1, out.numel(), device=DEV).view(out.shape)
        return (out * r).sum(), (pre > 0).detach()

    def grads(f, mask=None):
        for p in (conv.weight, bn.weight, bn.bias):
            p.grad = None
        h = head.to(DEV).requires_grad_(True)
        loss, m = f(h, mask)
        loss.backward()
        return [h.grad, conv.weight.grad.clone(), bn.weight.grad.clone(), bn.bias.grad.clone()], m

    got, mask = grads(torch.compile(chain, backend="inductor", fullgraph=True))
    want, _ = grads(chain, mask.float())
    for i, (a, b) in enumerate(zip(got, want)):
        assert float(b.norm()) > 0, i
        assert _nerr(a, b) < 2e-3, (i, _nerr(a, b))

# ==== C. the module and the training step, compiled with default settings =========================================================
@pytest.mark.parametrize("warped", [False, True], ids=["lift", "forward_warped"])
def test_compiled_module_matches_fp64(plain, warped):
    if warped:
        c = _make(NAME, 2, 2, seed=WARP_SEED)
        lift = LiftSplat.from_config(c["cfg"]).to(DEV)
        f = torch.compile(lambda h: lift.forward_warped(h, c["Kd"], c["Ed"], c["fd"], c["ext"]))
        h = c["hd"].clone().requires_grad_(True)
        bev = f(h)
        bev.backward(c["gd"].unflatten(0, (2, 2)))
        _assert_warped_bev(bev, c, _want_bev(c), "forward_warped")
        _assert_warped_grad(h.grad, c, _want_grad(c, c["gout"], "g"), c["gout"], "forward_warped")
        return
    lift = LiftSplat.from_config(CFG).to(DEV)
    f = torch.compile(lambda h: lift(h, plain["Kd"], plain["Ed"]))
    for _ in range(2):                                               # the second call runs the cached graph(s)
        h = plain["hd"].clone().requires_grad_(True)
        bev = f(h)
        bev.backward(plain["gd"])
        _assert_bev(bev, plain["exact"], "lift")
        _assert_grad(h.grad, plain["gexact"], "lift")

def test_compiled_training_step_matches_eager_and_fp64_replica():
    """LiftTrainer(precision=32) with model.forward compiled (the depth layer, a Python autograd.Function over the C ABI, breaks the
    graph): the flat gradient within 1e-5 of the eager step's, parameter by parameter, and within TRAIN_GRAD_TOL of the fp64 replica."""
    batch = synthetic_batch(TRAIN_CFG, 2, 2, DEV, seed=9, feature_input=True)
    eager = LiftTrainer(TRAIN_CFG, DEV, precision=32, feature_input=True, seed=3)
    comp = LiftTrainer(TRAIN_CFG, DEV, precision=32, feature_input=True, seed=3)
    comp.model.forward = torch.compile(comp.model.forward)
    loss_e, loss_c = float(eager.forward_backward(batch)), float(comp.forward_backward(batch))
    assert abs(loss_c - loss_e) <= 1e-5 * abs(loss_e), (loss_c, loss_e)
    _, want = _replica_loss_and_grads(comp.model, batch, True, TRAIN_CFG)
    fe, fc = eager.bucket.flat.detach().cpu(), comp.bucket.flat.detach().cpu()
    off = 0
    for k, p in comp.model.named_parameters():
        if not p.requires_grad:
            continue
        got, ref = fc[off:off + p.numel()], fe[off:off + p.numel()]
        off += p.numel()
        if want[k] is None:                                          # the image encoder: the step starts from features
            assert float(got.abs().max()) == 0 and float(ref.abs().max()) == 0, k
            continue
        assert float(ref.norm()) > 0, k
        assert _nerr(got, ref) < 1e-5, (k, _nerr(got, ref))
        assert O.normwise_error(got.view(p.shape), want[k]) < TRAIN_GRAD_TOL, k
    assert off == fc.numel()
