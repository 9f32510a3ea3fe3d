"""GPU: the fused BatchNorm3d (csrc/batch_norm.cu, torch.ops.fiery_b200.batch_norm_act, FusedBatchNorm3d, install.use_fused_batch_norm).

Every mode (train / eval x ReLU x residual x affine) against fp64 F.batch_norm (+ ReLU + add), each output within 3x of nn.BatchNorm3d's
own fp32 CUDA error; shapes around the 4096-pixel pieces, the channel and frame counts, strided and misaligned inputs and one tensor
past 2^31 elements; NaN-guarded outputs from a NaN-filled workspace; bit-reproducibility across calls, layouts, addresses and graph
replay; opcheck and torch.compile; whole TemporalModels with the four swaps (and with this one alone) against the fp64 oracle; and a
swapped step that dispatches no torch batch norm or ReLU on a map."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.utils._python_dispatch import TorchDispatchMode

from fiery_b200 import _lib, install, ops  # noqa: F401  (registers the operators)
from fiery_b200.batch_norm import FusedBatchNorm3d
from fiery_b200.batch_norm import backward as bn_backward
from fiery_b200.batch_norm import forward as bn_forward
from fiery_b200.temporal import temporal_model_forward
from oracle import temporal_oracle as TO
from tests._temporal_models import temporal_model

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
EPS = 1e-5


@pytest.fixture(autouse=True, scope="module")
def _no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _nerr(a, b):
    return TO.normwise_error(a, b)


def _data(shape, seed, affine=True):
    g = torch.Generator().manual_seed(seed)
    c = shape[1]
    x = (torch.randn(shape, generator=g) * 1.5 + torch.randn(c, generator=g).view(1, c, 1, 1, 1)).to(DEV)
    w = (torch.rand(c, generator=g) + 0.5).to(DEV) if affine else None
    b = (torch.rand(c, generator=g) - 0.5).to(DEV) if affine else None
    rm = (torch.randn(c, generator=g) * 0.5).to(DEV)
    rv = (torch.rand(c, generator=g) + 0.5).to(DEV)
    r = torch.randn(shape, generator=g).to(DEV)
    gy = torch.randn(shape, generator=g).to(DEV)
    return x, w, b, rm, rv, r, gy


def _torch_bn(x, w, b, rm, rv, r, gy, training, relu, dtype):
    """F.batch_norm (+ ReLU + add) in ``dtype``: (y, mean, var, running_mean, running_var, dx, dw, db)"""
    xi = x.detach().to(dtype).clone().requires_grad_(True)
    wi = w.detach().to(dtype).clone().requires_grad_(True) if w is not None else None
    bi = b.detach().to(dtype).clone().requires_grad_(True) if b is not None else None
    rmi, rvi = rm.to(dtype).clone(), rv.to(dtype).clone()
    y = F.batch_norm(xi, rmi, rvi, wi, bi, training, 0.1, EPS)
    if relu:
        y = F.relu(y)
    if r is not None:
        y = y + r.to(dtype)
    y.backward(gy.to(dtype))
    dims = (0, 2, 3, 4)
    xd = x.to(dtype)
    mean, var = (xd.mean(dims), xd.var(dims, unbiased=False)) if training else (rm.to(dtype), rv.to(dtype))
    return (y.detach(), mean, var, rmi, rvi, xi.grad, wi.grad if wi is not None else None, bi.grad if bi is not None else None)


def _fused(x, w, b, rm, rv, r, gy, training, relu):
    """the module and the operator: the same eight results"""
    bn = nn.BatchNorm3d(x.shape[1], eps=EPS, affine=w is not None).to(DEV).train(training)
    with torch.no_grad():
        if w is not None:
            bn.weight.copy_(w)
            bn.bias.copy_(b)
        bn.running_mean.copy_(rm)
        bn.running_var.copy_(rv)
    f = FusedBatchNorm3d(bn)
    xi = x.detach().clone().requires_grad_(True)
    y = f.forward_act(xi, relu, r)
    y.backward(gy)
    _, mean, var = torch.ops.fiery_b200.batch_norm_act(x, w, b, None if training else rm, None if training else rv, r, training, EPS,
                                                       relu)
    return (y.detach(), mean, var, f.running_mean, f.running_var, xi.grad, f.weight.grad if w is not None else None,
            f.bias.grad if w is not None else None)


NAMES = ("y", "mean", "var", "running_mean", "running_var", "dx", "dweight", "dbias")


@pytest.mark.parametrize("affine", [True, False], ids=["affine", "plain"])
@pytest.mark.parametrize("residual", [True, False], ids=["res", "nores"])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "norelu"])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_every_mode_against_fp64(training, relu, residual, affine):
    x, w, b, rm, rv, r, gy = _data((2, 35, 3, 52, 48), seed=1, affine=affine)
    r = r if residual else None
    want = _torch_bn(x, w, b, rm, rv, r, gy, training, relu, torch.float64)
    theirs = _torch_bn(x, w, b, rm, rv, r, gy, training, relu, torch.float32)
    got = _fused(x, w, b, rm, rv, r, gy, training, relu)
    for name, a, t, e in zip(NAMES, got, theirs, want):
        if e is None:
            assert a is None, name
            continue
        err, bar = _nerr(a, e), max(3 * _nerr(t, e), 1e-6)
        assert err <= bar, f"{name}: {err:.3e} (torch fp32 {_nerr(t, e):.3e})"


# (b, C, s, X, Y): X*Y at and around the 4096-pixel pieces, one and several pieces per plane; C 1..128; b*s 1..12
SHAPES = [(2, 3, 1, 1, 3), (1, 32, 3, 1, 3), (4, 35, 3, 2, 2), (1, 64, 2, 1, 4095), (3, 1, 1, 64, 64), (1, 35, 5, 1, 4097),
          (2, 128, 1, 8, 1023), (1, 64, 12, 200, 200), (3, 35, 3, 200, 400), (6, 32, 2, 4, 4), (1, 1, 1, 2, 8193),
          (2, 64, 3, 5, 5), (12, 35, 1, 3, 3), (4, 35, 3, 1, 1)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_shapes_against_fp64(shape, training):
    x, w, b, rm, rv, r, gy = _data(shape, seed=sum(shape))
    want = _torch_bn(x, w, b, rm, rv, r, gy, training, True, torch.float64)
    theirs = _torch_bn(x, w, b, rm, rv, r, gy, training, True, torch.float32)
    got = _fused(x, w, b, rm, rv, r, gy, training, True)
    for name, a, t, e in zip(NAMES, got, theirs, want):
        err, bar = _nerr(a, e), max(3 * _nerr(t, e), 1e-6)
        assert err <= bar, f"{name}: {err:.3e} (torch fp32 {_nerr(t, e):.3e})"


def _op_all(x, w, b, r, gy, training=True, relu=True, rm=None, rv=None):
    y, mean, var = bn_forward(x, w, b, rm, rv, r, training, EPS, relu)
    dx, dw, db = bn_backward(gy, x, w, b, mean, var, training, EPS, relu, True, True, True)
    return y, mean, var, dx, dw, db


def _layouts(x):
    """x's values laid out as the permuted (b, s, C, X, Y) tensor, a channel slice and a 4-byte-misaligned copy"""
    b, c, s, h, w = x.shape
    perm = x.permute(0, 2, 1, 3, 4).contiguous().permute(0, 2, 1, 3, 4)
    big = torch.full((b, c + 5, s, h, w), float("nan"), device=DEV)
    big[:, 3:3 + c] = x
    flat = torch.full((x.numel() + 1,), float("nan"), device=DEV)
    mis = flat[1:].view(x.shape)
    mis.copy_(x)
    return {"permuted": perm, "sliced": big[:, 3:3 + c], "misaligned": mis}


@pytest.mark.parametrize("grid", [(52, 48), (3, 5), (64, 64), (1, 4097)])
def test_layouts_and_addresses_bit_identical(grid):
    x, w, b, rm, rv, r, gy = _data((2, 35, 3, *grid), seed=5)
    for training in (True, False):
        ref = _op_all(x, w, b, r, gy, training, True, rm, rv)
        again = _op_all(x, w, b, r, gy, training, True, rm, rv)
        assert all(torch.equal(a, e) for a, e in zip(again, ref))
        for name, xl in _layouts(x).items():
            got = _op_all(xl, w, b, r, gy, training, True, rm, rv)
            assert all(torch.equal(a, e) for a, e in zip(got, ref)), name
        # the same values one element further on in every tensor: misaligned residual, gradient and outputs
        sh = lambda t: _layouts(t)["misaligned"]                        # noqa: E731
        got = _op_all(sh(x), w, b, sh(r), sh(gy), training, True, rm, rv)
        assert all(torch.equal(a, e) for a, e in zip(got, ref)), "all misaligned"


def test_guarded_outputs_and_nan_workspace():
    lib = _lib.load()
    for shape, relu, res in [((2, 35, 3, 52, 48), True, True), ((1, 3, 2, 3, 5), False, True), ((2, 4, 1, 1, 4097), True, False)]:
        x, w, b, rm, rv, r, gy = _data(shape, seed=9)
        n, c = x.numel(), shape[1]
        for training in (1, 0):
            ref = _op_all(x, w, b, r if res else None, gy, bool(training), relu, rm, rv)
            d = _lib.BatchNormDesc()
            d.batch, d.channels, d.frames, d.pixels = shape[0], c, shape[2], shape[3] * shape[4]
            d.stride_b, d.stride_c, d.stride_t = x.stride(0), x.stride(1), x.stride(2)
            d.training, d.relu, d.eps = training, int(relu), EPS
            ws = torch.full((int(lib.fiery_batch_norm_workspace_bytes(d)) // 4 + 4,), float("nan"), device=DEV)
            yb = torch.full((n + 65,), float("nan"), device=DEV)
            mb, vb = torch.full((c + 64,), float("nan"), device=DEV), torch.full((c + 64,), float("nan"), device=DEV)
            _lib.call("fiery_batch_norm_forward", DEV, d, x.data_ptr(), w.data_ptr(), b.data_ptr(), rm.data_ptr(), rv.data_ptr(),
                      r.data_ptr() if res else 0, yb[33:].data_ptr(), mb[32:].data_ptr(), vb[32:].data_ptr(), ws.data_ptr())
            assert torch.equal(yb[33:33 + n].view(shape), ref[0]) and torch.equal(mb[32:32 + c], ref[1])
            assert torch.equal(vb[32:32 + c], ref[2])
            for t, k in ((yb, 33), (mb, 32), (vb, 32)):
                assert torch.isnan(t[:k]).all() and torch.isnan(t[t.numel() - 32:]).all()
            ws.fill_(float("nan"))
            gb = torch.full((n + 65,), float("nan"), device=DEV)
            wb, bb = torch.full((c + 64,), float("nan"), device=DEV), torch.full((c + 64,), float("nan"), device=DEV)
            _lib.call("fiery_batch_norm_backward", DEV, d, x.data_ptr(), gy.data_ptr(), w.data_ptr(), b.data_ptr(), ref[1].data_ptr(),
                      ref[2].data_ptr(), gb[33:].data_ptr(), wb[32:].data_ptr(), bb[32:].data_ptr(), ws.data_ptr())
            assert torch.equal(gb[33:33 + n].view(shape), ref[3])
            assert torch.equal(wb[32:32 + c], ref[4]) and torch.equal(bb[32:32 + c], ref[5])
            for t, k in ((gb, 33), (wb, 32), (bb, 32)):
                assert torch.isnan(t[:k]).all() and torch.isnan(t[t.numel() - 32:]).all()


def test_one_value_per_channel_in_training_raises():
    x = torch.randn(1, 4, 1, 1, 1, device=DEV)
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        torch.ops.fiery_b200.batch_norm_act(x, None, None, None, None, None, True, EPS, True)
    f = FusedBatchNorm3d(nn.BatchNorm3d(4).to(DEV))
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        f(x)
    f.eval()
    y = f(x)                                                            # eval takes one value
    assert torch.allclose(y, (x - f.running_mean.view(1, 4, 1, 1, 1)) / (1 + EPS) ** 0.5, atol=1e-6)


def test_graph_replay_bit_identical():
    x, w, b, rm, rv, r, gy = _data((3, 35, 3, 52, 48), seed=4)
    ref = _op_all(x, w, b, r, gy)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _op_all(x, w, b, r, gy)                                         # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = _op_all(x, w, b, r, gy)
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, e) for a, e in zip(out, ref))


def test_module_step_captures_in_a_graph():
    """forward, backward and the running-statistics update of a FusedBatchNorm3d under graph capture, against eager steps"""
    x, *_ , gy = _data((2, 35, 3, 52, 48), seed=6)
    eager = FusedBatchNorm3d(nn.BatchNorm3d(35, momentum=None).to(DEV))
    graphed = copy.deepcopy(eager)
    xi = x.clone().requires_grad_(True)

    def step(m):
        y = m.forward_act(xi, True)
        y.backward(gy)
        return y

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(copy.deepcopy(eager))
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg = step(graphed)
    graphed.num_batches_tracked.zero_()
    graphed.running_mean.zero_()
    graphed.running_var.fill_(1)
    for _ in range(3):
        graph.replay()
        ye = step(eager)
    torch.cuda.synchronize()
    assert torch.equal(yg, ye)
    for (n, a), (_, e) in zip(graphed.named_buffers(), eager.named_buffers()):
        assert torch.equal(a, e), n


def test_past_2_31_elements():
    if torch.cuda.get_device_properties(DEV).total_memory < 40 << 30:
        pytest.skip("needs about 30 GB of device memory")
    shape = (1, 4, 1, 23200, 23200)                                      # 2.15e9 elements: offsets past 2^31
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(shape, device=DEV, generator=g)
    x[:, 1] += 3.0
    w = torch.tensor([1.0, 0.5, 2.0, 1.5], device=DEV)
    b = torch.tensor([0.1, -0.2, 0.0, 0.3], device=DEV)
    y, mean, var = bn_forward(x, w, b, None, None, None, True, EPS, True)
    mean64 = torch.stack([x[:, c].double().mean() for c in range(4)])
    var64 = torch.stack([x[:, c].double().var(unbiased=False) for c in range(4)])
    assert torch.allclose(mean.double(), mean64, atol=1e-6) and torch.allclose(var.double(), var64, rtol=1e-6)
    scale = w.double() / (var.double() + EPS).sqrt()
    shift = b.double() - mean.double() * scale
    tail = x[0, :, 0, -1, -64:].double()                                   # the last pixels of every channel
    want = (scale[:, None] * tail + shift[:, None]).clamp_min(0)
    assert torch.allclose(y[0, :, 0, -1, -64:].double(), want, atol=1e-5)
    del y
    dx, dw, db = bn_backward(x, x, w, b, mean, var, True, EPS, True, True, True, True)   # grad_y = x: any values do
    m = (scale[:, None] * tail + shift[:, None]) > 0
    gm = torch.where(m, tail, 0)
    s1 = torch.stack([torch.where(x[:, c] * float(scale[c]) + float(shift[c]) > 0, x[:, c], 0).double().sum() for c in range(4)])
    assert torch.allclose(db.double(), s1, rtol=1e-5)
    n = x[0, 0].numel()
    s2 = dw.double() * (var.double() + EPS).sqrt()
    want_dx = scale[:, None] * (gm - s1[:, None] / n - (tail - mean.double()[:, None]) * s2[:, None] / (n * (var.double()[:, None] + EPS)))
    assert torch.allclose(dx[0, :, 0, -1, -64:].double(), want_dx, atol=1e-5, rtol=1e-5)


# ------------------------------------------------------------------------------------------------------------------------------
# operator checks
# ------------------------------------------------------------------------------------------------------------------------------
def test_opcheck():
    x, w, b, rm, rv, r, _ = _data((2, 6, 3, 4, 8), seed=2)
    xg, wg, bg = x.requires_grad_(True), w.requires_grad_(True), b.requires_grad_(True)
    for args in [(xg, wg, bg, None, None, r.requires_grad_(True), True, EPS, True), (xg, None, None, None, None, None, True, EPS, False),
                 (xg, wg, bg, rm, rv, None, False, EPS, True)]:
        torch.library.opcheck(torch.ops.fiery_b200.batch_norm_act.default, args)


def test_autocast_widens_and_returns_fp32():
    x, w, b, rm, rv, r, gy = _data((2, 35, 3, 8, 8), seed=7)
    xh = x.half().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16):
        y, _, _ = torch.ops.fiery_b200.batch_norm_act(xh, w, b, None, None, r.half(), True, EPS, True)
    assert y.dtype == torch.float32
    y.backward(gy)
    ref = _op_all(xh.detach().float(), w, b, r.half().float(), gy)
    assert torch.equal(y.detach(), ref[0]) and xh.grad.dtype == torch.float16
    assert torch.equal(xh.grad, ref[3].half())


@pytest.mark.parametrize("backend", ["aot_eager", "inductor"])
def test_compiled_forward_backward(backend):
    x, w, b, rm, rv, r, gy = _data((2, 35, 3, 16, 12), seed=8)
    eager = FusedBatchNorm3d(nn.BatchNorm3d(35).to(DEV))
    comp = copy.deepcopy(eager)

    def run(m, fn):
        xi, ri = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
        y = fn(xi, ri)
        y.backward(gy)
        return y.detach(), xi.grad, ri.grad, m.weight.grad, m.bias.grad

    ref = run(eager, lambda xi, ri: eager.forward_act(xi, True, ri))
    fn = torch.compile(lambda xi, ri: comp.forward_act(xi, True, ri), backend=backend, fullgraph=True)
    got = run(comp, fn)
    assert all(torch.equal(a, e) for a, e in zip(got, ref))
    for (n, a), (_, e) in zip(comp.named_buffers(), eager.named_buffers()):
        assert torch.allclose(a.double(), e.double(), rtol=1e-6, atol=1e-7), n


def test_frozen_inputs_launch_only_what_is_asked(monkeypatch):
    calls = []
    real = bn_backward

    def spy(*args):
        calls.append(tuple(args[-3:]))
        return real(*args)

    monkeypatch.setattr("fiery_b200.batch_norm.backward", spy)
    x, w, b, _, _, r, gy = _data((2, 6, 3, 4, 8), seed=3)
    for need_x, need_w, need_r in [(True, False, False), (False, True, False), (False, False, True), (True, True, True)]:
        calls.clear()
        xi, wi, bi, ri = x.clone().requires_grad_(need_x), w.clone().requires_grad_(need_w), b.clone().requires_grad_(need_w), \
            r.clone().requires_grad_(need_r)
        y, _, _ = torch.ops.fiery_b200.batch_norm_act(xi, wi, bi, None, None, ri, True, EPS, True)
        y.backward(gy)
        assert calls == ([(need_x, need_w, need_w)] if need_x or need_w else [])
        assert (xi.grad is not None) == need_x and (wi.grad is not None) == need_w and (ri.grad is not None) == need_r
        if need_r:
            assert torch.equal(ri.grad, gy)


# ------------------------------------------------------------------------------------------------------------------------------
# whole TemporalModel
# ------------------------------------------------------------------------------------------------------------------------------
GRID = (52, 48)


def _model(rf, inbetween, seed=0, grid=GRID):
    torch.manual_seed(seed)
    m = temporal_model(70, rf, grid, start_out_channels=64, inbetween_layers=inbetween)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm3d):
            mod.weight.data.uniform_(0.5, 1.5)
            mod.bias.data.uniform_(-0.2, 0.2)
            mod.running_mean.uniform_(-0.1, 0.1)
            mod.running_var.uniform_(0.5, 1.5)
    return m.to(DEV)


def _swapped(m, swaps):
    s = copy.deepcopy(m)
    h = type("M", (), {"temporal_model": s})()
    if swaps == "all":
        install.use_tensor_core_temporal_model(h)
        install.use_tensor_core_causal_convs(h)
        install.use_tensor_core_pyramid_pooling(h)
    install.use_fused_batch_norm(h)
    assert any(isinstance(x, FusedBatchNorm3d) for x in s.modules())
    return s


def _step(m, bev, ego, gout, route, amp=False, tf32=False):
    bev = bev.detach().clone().requires_grad_(True)
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            y = temporal_model_forward(m, bev, ego) if route == "folded" else m(TO.egopose_concat(bev, ego.to(bev.dtype)))
        out = y if y.dtype == torch.float64 else y.float()
        out.backward(gout.to(out.dtype))
    finally:
        torch.backends.cudnn.allow_tf32 = False
    return out.detach(), bev.grad, {n: p.grad.detach().clone() for n, p in m.named_parameters()}


MODEL_CASES = [(rf, inb, swaps, route) for rf, inb in ((3, 0), (5, 0), (3, 1)) for swaps, route in
               (("all", "concat"), ("all", "folded"), ("bn", "concat"))]


@pytest.mark.parametrize("amp", [False, True], ids=["fp32", "amp"])
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("rf,inbetween,swaps,route", MODEL_CASES, ids=lambda v: str(v))
def test_whole_model_matches_oracle(rf, inbetween, swaps, route, train, amp):
    ref = _model(rf, inbetween)
    sw = _swapped(ref, swaps)
    ref64 = copy.deepcopy(ref).double()
    for m in (ref, sw, ref64):
        m.train(train)
    gen = torch.Generator().manual_seed(11 + rf)
    s = rf
    bev = torch.randn((2, s, 64, *GRID), generator=gen).to(DEV)
    ego = torch.randn((2, s, 6), generator=gen).to(DEV)
    gout = torch.randn((2, 1, 64, *GRID), generator=gen).to(DEV)
    y64, gx64, gp64 = _step(ref64, bev.double(), ego.double(), gout.double(), "concat")
    y0, gx0, gp0 = _step(ref, bev, ego, gout, "concat", amp, tf32=True)
    y1, gx1, gp1 = _step(sw, bev, ego, gout, route, amp)
    assert set(gp1) == set(gp0) == set(gp64)
    for what, a, r, o in [("out", y1, y64, y0), ("grad_bev", gx1, gx64, gx0)] + [(n, gp1[n], gp64[n], gp0[n]) for n in gp64]:
        err, bar = _nerr(a, r), max(3 * _nerr(o, r), 1e-5)
        assert err <= bar, f"{what}: {err:.3e} vs oracle {_nerr(o, r):.3e}"
    # the running statistics after the step: the batch statistics of TF32 tensor-core outputs in the swapped model, so against the
    # fp32 reference's within the bar of tests/test_temporal_tail_gpu.py
    for (n, b1), (_, b0) in zip(sw.named_buffers(), ref.named_buffers()):
        if b1.dtype.is_floating_point:
            assert _nerr(b1, b0) < 1e-3, n
        else:
            assert torch.equal(b1, b0), n


class _Recorder(TorchDispatchMode):
    def __init__(self):
        super().__init__()
        self.ops = []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        self.ops.append((str(func.overloadpacket.__name__), args))
        return out


def test_swapped_step_dispatches_no_torch_batch_norm_or_relu_on_a_map():
    grid = (200, 200)
    ref = _model(3, 0, seed=1, grid=grid)
    sw = _swapped(ref, "all").train(True)
    gen = torch.Generator().manual_seed(2)
    bev = torch.randn((3, 3, 64, *grid), generator=gen).to(DEV).requires_grad_(True)
    ego = torch.randn((3, 3, 6), generator=gen).to(DEV)
    with _Recorder() as rec:
        y = temporal_model_forward(sw, bev, ego)
        y.sum().backward()
    names = [n for n, _ in rec.ops]
    assert "batch_norm_act" in names and "batch_norm_act_backward" in names
    for n, args in rec.ops:
        maps = [a for a in args if isinstance(a, torch.Tensor) and a.dim() == 5 and tuple(a.shape[3:]) == grid]
        if not maps:
            continue
        assert not ("batch_norm" in n and not n.startswith("batch_norm_act")), n
        assert n not in ("relu", "relu_", "threshold_backward", "clamp_min", "clamp_min_"), n
