"""GPU: the temporal model's causal convolutions (fiery_b200/csrc/causal_conv.cu, fiery_b200/causal_conv.py) -- forward, input gradient
and weight gradient against fp64 F.conv3d on the causally padded input, the weight gradient's reproducibility, whole TemporalModels with
both tensor-core swaps against the oracle (oracle/temporal_oracle.py), the fallback for maps the TMA cannot take, and the operators
under opcheck, aot_eager and inductor.

Parity bar (the first BEV convolution's, tests/test_first_conv_backward_gpu.py): TF32 operands and fp32 accumulation against fp64 --
normwise < 1e-3, and within 3x of the larger of cuDNN TF32's error and the error of fp64 on TF32-rounded operands.  Small integers are
exact in TF32 and fp32, so on them every output and gradient must be bit-exact."""
import copy

import pytest
import torch
import torch.nn.functional as F

from fiery_b200 import _lib, install, ops  # noqa: F401
from fiery_b200.causal_conv import TensorCoreCausalConv3d, conv_backward_data, conv_backward_weight, conv_forward
from fiery_b200.geometry import _stream_ptr
from fiery_b200.temporal import TensorCoreTemporalBlock, temporal_model_forward
from oracle import temporal_oracle as TO
from tests._temporal_models import temporal_model

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
CHANNELS = [(35, 35), (32, 32), (64, 64), (1, 8), (35, 64)]
GRIDS = [(1, 4), (3, 4), (7, 12), (52, 48), (200, 200), (400, 200)]
# every (channels, grid) pair with both kt; frames and batch cycle so each value meets every grid; the two largest grids keep b * s small
CASES = [(kt, ch, grid, (1, 3)[(i + j) % 2] if j < 4 else 1, (1, 2, 3, 5)[(i + j + kt) % 4] if j < 4 else (1, 2)[(i + kt) % 2])
         for kt in (1, 2) for i, ch in enumerate(CHANNELS) for j, grid in enumerate(GRIDS)]


@pytest.fixture(autouse=True, scope="module")
def _no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _nerr(a, b):
    return TO.normwise_error(a, b)


def _tensors(kt, cin, cout, grid, b, s, seed, ints=True):
    gen = torch.Generator().manual_seed(seed)
    mk = (lambda *shape: torch.randint(-2, 3, shape, generator=gen).float()) if ints else (lambda *shape: torch.randn(shape, generator=gen))
    x = mk(b, cin, s, *grid).to(DEV)
    w = mk(cout, cin, kt, 3, 3).to(DEV)
    if not ints:
        w = w / (cin * 9 * kt) ** 0.5
    gy = mk(b, cout, s, *grid).to(DEV)
    return x, w, gy


def _reference(x, w, gy, dtype=torch.float64):
    """F.conv3d on the causally padded input (the reference CausalConv3d's pad + conv) and its gradients, in dtype"""
    kt = w.shape[2]
    xd = x.to(dtype).detach().requires_grad_(True)
    wd = w.to(dtype).detach().requires_grad_(True)
    y = F.conv3d(F.pad(xd, (1, 1, 1, 1, kt - 1, 0)), wd)
    y.backward(gy.to(dtype))
    return y.detach(), xd.grad, wd.grad


@pytest.mark.parametrize("kt,ch,grid,b,s", CASES, ids=lambda v: str(v).replace(" ", ""))
def test_small_integers_bit_exact(kt, ch, grid, b, s):
    """Forward, input gradient and weight gradient equal fp64 exactly.  The outputs and the workspace start NaN-filled (deterministic
    mode fills uninitialised memory), so an element a kernel does not write shows up; frame 0 pins the causal padding in front and the
    last frame the input gradient's zero beyond it."""
    cin, cout = ch
    x, w, gy = _tensors(kt, cin, cout, grid, b, s, seed=CASES.index((kt, ch, grid, b, s)))
    y_ref, gx_ref, gw_ref = _reference(x, w, gy)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        y = conv_forward(x, w)
        gx = conv_backward_data(gy, tuple(x.shape), w)
        gw = conv_backward_weight(gy, x, w)
    finally:
        torch.use_deterministic_algorithms(old)
    assert y.is_contiguous() and torch.equal(y.double(), y_ref)
    assert torch.equal(gx.double(), gx_ref)
    assert torch.equal(gw.double(), gw_ref)


def _tf32(t):
    """round to TF32 (nearest, ties away), as cvt.rna does"""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).view(t.shape)


@pytest.mark.parametrize("kt", [1, 2])
@pytest.mark.parametrize("ch", [(35, 35), (32, 32), (64, 64)])
@pytest.mark.parametrize("grid", [(52, 48), (200, 200)])
def test_random_fp32_against_fp64_and_cudnn(kt, ch, grid):
    cin, cout = ch
    x, w, gy = _tensors(kt, cin, cout, grid, 3, 3, seed=7, ints=False)
    ref = _reference(x, w, gy)
    got = (conv_forward(x, w), conv_backward_data(gy, tuple(x.shape), w), conv_backward_weight(gy, x, w))
    torch.backends.cudnn.allow_tf32 = True
    try:
        tf = _reference(x, w, gy, torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32 = False
    rr = _reference(_tf32(x), _tf32(w), _tf32(gy))
    for what, g_, r_, t_, q_ in zip(("forward", "grad_x", "grad_w"), got, ref, tf, rr):
        err = _nerr(g_, r_)
        bar = 3 * max(_nerr(t_, r_), _nerr(q_, r_))
        assert err < 1e-3 and err <= bar, f"{what}: {err:.3e} (bar {bar:.3e})"


def test_weight_gradient_reproducible_eager_and_graph_replay():
    """The same bits whatever the workspace held before, run to run and under graph replay."""
    from fiery_b200.causal_conv import _desc
    x, w, gy = _tensors(2, 35, 35, (200, 200), 3, 3, seed=3, ints=False)
    lib = _lib.load()
    d = _desc(tuple(x.shape), 35, 2)
    need = int(lib.fiery_causal_conv3d_backward_weight_workspace_bytes(d))

    def run(fill):
        ws = torch.full((need // 4,), fill, dtype=torch.float32, device=DEV)
        gw = torch.full_like(w, float("nan"))
        _lib.check(lib.fiery_causal_conv3d_backward_weight(d, x.data_ptr(), gy.data_ptr(), gw.data_ptr(), ws.data_ptr(),
                                                           _stream_ptr(DEV)), "backward_weight")
        return gw

    first = run(float("nan"))
    for fill in (0.0, 1e30, -3.0):
        assert torch.equal(run(fill), first)
    assert torch.equal(conv_backward_weight(gy, x, w), first)
    conv_forward(x, w)                                        # pack cached before capture
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        conv_backward_weight(gy, x, w)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = conv_forward(x, w)
        gw = conv_backward_weight(gy, x, w)
    y0 = conv_forward(x, w)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(gw, first) and torch.equal(y, y0)


def test_zero_frames():
    x, w, gy = _tensors(2, 35, 32, (8, 8), 1, 1, seed=1)
    assert tuple(conv_forward(x[:0], w).shape) == (0, 32, 1, 8, 8)
    assert tuple(conv_forward(x[:, :, :0], w).shape) == (1, 32, 0, 8, 8)
    assert torch.count_nonzero(conv_backward_weight(gy[:0], x[:0], w)) == 0


def test_noncontiguous_and_half_inputs_are_read_as_fp32():
    x, w, gy = _tensors(2, 35, 35, (52, 48), 2, 3, seed=4)
    want = conv_forward(x, w)
    assert torch.equal(conv_forward(x.half(), w), want)                              # small integers are exact in fp16
    xt = x.permute(0, 2, 1, 3, 4).contiguous().permute(0, 2, 1, 3, 4)               # frame-major storage
    assert not xt.is_contiguous() and torch.equal(conv_forward(xt, w), want)


def test_uncovered_map_width_falls_back_with_one_warning():
    torch.manual_seed(0)
    ref = TO.CausalConv3d(35, 35).to(DEV).eval()
    tc = TensorCoreCausalConv3d.from_module(ref)
    x = torch.randn(2, 35, 3, 9, 10, device=DEV)
    with pytest.warns(RuntimeWarning, match="Y = 10"):
        got = tc(x)
    assert torch.equal(got, TO.CausalConv3d.forward(ref, x))


# ------------------------------------------------------------------------------------------------------------------------------
# whole temporal models
# ------------------------------------------------------------------------------------------------------------------------------
def _model(grid, rf=3, inbetween=0, seed=0):
    torch.manual_seed(seed)
    m = temporal_model(70, rf, grid, start_out_channels=64, inbetween_layers=inbetween)
    for mod in m.modules():                                   # non-trivial BN affine / running statistics
        if isinstance(mod, torch.nn.BatchNorm3d):
            mod.weight.data.uniform_(0.5, 1.5)
            mod.bias.data.uniform_(-0.2, 0.2)
            mod.running_mean.uniform_(-0.1, 0.1)
            mod.running_var.uniform_(0.5, 1.5)
    return m.to(DEV)


def _swapped(m):
    s = copy.deepcopy(m)
    holder = type("M", (), {"temporal_model": s})()
    install.use_tensor_core_temporal_model(holder)
    install.use_tensor_core_causal_convs(holder)
    assert all(isinstance(b, TensorCoreTemporalBlock) for b in s.model if "TemporalBlock" in type(b).__name__)
    causal = [x for x in s.modules() if isinstance(x, (TO.CausalConv3d, TensorCoreCausalConv3d))]
    assert causal and all(isinstance(x, TensorCoreCausalConv3d) for x in causal)
    return s


def _run(m, bev, ego, gout, route, amp=False, tf32=False):
    """outputs, BEV gradient and parameter gradients of one step; route "folded": temporal_model_forward, "concat": the egopose
    concat and the model's own forward.  tf32: cuDNN may use TF32 (the oracle's bar)"""
    bev = bev.detach().clone().requires_grad_(True)
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            y = temporal_model_forward(m, bev, ego) if route == "folded" else m(TO.egopose_concat(bev, ego))
        y.float().backward(gout)
    finally:
        torch.backends.cudnn.allow_tf32 = False
    return y.float().detach(), bev.grad, {n.replace("_orig_mod.", ""): p.grad.detach().clone() for n, p in m.named_parameters()}


@pytest.mark.parametrize("route", ["folded", "concat"])
@pytest.mark.parametrize("amp", [False, True], ids=["fp32", "amp"])
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("rf,inbetween", [(3, 0), (5, 0), (3, 1)], ids=["rf3", "rf5", "rf3_inbetween1"])
def test_whole_model_matches_oracle(rf, inbetween, train, amp, route):
    """Both swaps against fp64, within 3x of the oracle's own error with cuDNN in TF32 (fp32) or under the same autocast (amp) --
    the bars of test_temporal_entry_gpu.py::test_whole_model_matches_oracle -- or within 3x of the error of the same model with the
    temporal-entry swap alone.  The second bar is for the deeper models in eval mode: there a few BatchNorm weight gradients of the
    later blocks (sums of gradient x normalised activation that nearly cancel) carry 3-4x the oracle's error with either swap, since
    the tensor-core paths truncate or round every activation to TF32 where cuDNN keeps some of its operands in fp32; the causal
    convolutions must add nothing beyond what the entry swap already does."""
    grid = (52, 48)
    ref = _model(grid, rf, inbetween)
    sw = _swapped(ref)
    entry = copy.deepcopy(ref)
    install.use_tensor_core_temporal_model(type("M", (), {"temporal_model": entry})())
    ref64 = copy.deepcopy(ref).double()
    for m in (ref, sw, entry, ref64):
        m.train(train)
    gen = torch.Generator().manual_seed(11)
    bev = torch.randn((2, rf, 64, *grid), generator=gen).to(DEV)
    ego = torch.randn((2, rf, 6), generator=gen).to(DEV)
    gout = torch.randn((2, 1, 64, *grid), generator=gen).to(DEV)
    y64, gx64, gp64 = _run(ref64, bev.double(), ego.double(), gout.double(), "concat")
    y0, gx0, gp0 = _run(ref, bev, ego, gout, "concat", amp, tf32=True)
    y1, gx1, gp1 = _run(sw, bev, ego, gout, route, amp)
    y2, gx2, gp2 = _run(entry, bev, ego, gout, route, amp)
    assert set(gp1) == set(gp0) == set(gp64)
    for what, a, r, o, e in [("out", y1, y64, y0, y2), ("grad_bev", gx1, gx64, gx0, gx2)] + \
            [(n, gp1[n], gp64[n], gp0[n], gp2[n]) for n in gp64]:
        err, bar = _nerr(a, r), max(3 * _nerr(o, r), 3 * _nerr(e, r), 1e-5)
        assert err <= bar, f"{what}: {err:.3e} vs oracle {_nerr(o, r):.3e}, entry swap alone {_nerr(e, r):.3e}"
    if train:                                                   # running statistics follow the same batches
        for (n, b1), (_, b0) in zip(sw.named_buffers(), ref.named_buffers()):
            if b1.dtype.is_floating_point:
                assert _nerr(b1, b0) < 1e-3, n


# ------------------------------------------------------------------------------------------------------------------------------
# operators under the compiler
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kt", [1, 2])
def test_opcheck(kt):
    x, w, gy = _tensors(kt, 35, 32, (8, 8), 2, 3, seed=9, ints=False)
    torch.library.opcheck(torch.ops.fiery_b200.causal_conv3d.default, (x.requires_grad_(True), w.requires_grad_(True)))
    for ni, nw in ((True, True), (True, False), (False, True)):
        torch.library.opcheck(torch.ops.fiery_b200.causal_conv3d_backward.default, (gy, x.detach(), w.detach(), ni, nw))


@pytest.mark.parametrize("backend", ["aot_eager", "inductor"])
def test_compiled_model_matches_eager(backend):
    grid = (52, 48)
    ref = _model(grid, seed=6)
    sw = _swapped(ref).train(True)
    comp = copy.deepcopy(sw)
    gen = torch.Generator().manual_seed(8)
    bev = torch.randn((2, 3, 64, *grid), generator=gen).to(DEV)
    ego = torch.randn((2, 3, 6), generator=gen).to(DEV)
    gout = torch.randn((2, 1, 64, *grid), generator=gen).to(DEV)
    y64, gx64, gp64 = _run(copy.deepcopy(ref).double().train(True), bev.double(), ego.double(), gout.double(), "concat")
    y0, gx0, gp0 = _run(sw, bev, ego, gout, "concat")
    fn = torch.compile(comp, backend=backend, fullgraph=True)
    y1, gx1, gp1 = _run(fn, bev, ego, gout, "concat")
    assert set(gp1) == set(gp0)
    for what, a, e, r in [("out", y1, y0, y64), ("grad_bev", gx1, gx0, gx64)] + [(n, gp1[n], gp0[n], gp64[n]) for n in gp0]:
        assert _nerr(a, r) <= max(1.5 * _nerr(e, r), 1e-5), f"{what}: compiled {_nerr(a, r):.3e} eager {_nerr(e, r):.3e}"


def test_frozen_weights_launch_no_weight_gradient(monkeypatch):
    """needs_input_grad decides which gradients run: frozen weights launch no weight gradient, a frozen input no input gradient."""
    from fiery_b200 import causal_conv
    calls = []
    for name in ("conv_backward_data", "conv_backward_weight"):
        monkeypatch.setattr(causal_conv, name, (lambda f, n: lambda *a, **k: calls.append(n) or f(*a, **k))(getattr(causal_conv, name), name))
    x, w, gy = _tensors(2, 35, 35, (8, 8), 1, 3, seed=2, ints=False)
    for need_x, need_w, want in ((True, False, ["conv_backward_data"]), (False, True, ["conv_backward_weight"]),
                                 (True, True, ["conv_backward_data", "conv_backward_weight"])):
        calls.clear()
        xi = x.detach().requires_grad_(need_x)
        wi = w.detach().requires_grad_(need_w)
        torch.ops.fiery_b200.causal_conv3d(xi, wi).backward(gy)
        assert calls == want
        assert (xi.grad is not None) == need_x and (wi.grad is not None) == need_w
