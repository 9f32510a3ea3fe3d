"""GPU: the temporal block's fused 1x1x1 input projections (fiery_b200/csrc/temporal_entry.cu, fiery_b200/temporal.py) -- forward,
input gradient and weight gradient against fp64, the folded egopose route, TensorCoreTemporalBlock inside a whole TemporalModel
(oracle/temporal_oracle.py) in train and eval, fp32 and autocast, the lift -> warp -> temporal model chain, and the operators under
opcheck, aot_eager and inductor.

Parity bar (the first BEV convolution's, tests/test_first_conv_backward_gpu.py): TF32 operands and fp32 accumulation against fp64 --
normwise < 1e-3, and within 3x of the larger of cuDNN TF32's error and the error of fp64 on TF32-rounded operands.  Small integers are
exact in TF32 and fp32, so on them every output and gradient must be bit-exact."""
import copy

import pytest
import torch
import torch.nn.functional as F

from fiery_b200 import ops  # noqa: F401  (registers the operators)
from fiery_b200 import install
from fiery_b200.temporal import TensorCoreTemporalBlock, entry_backward_data, entry_backward_weight, entry_forward, \
    temporal_model_forward
from oracle import temporal_oracle as TO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GRIDS = [(2, 2), (8, 8), (52, 49), (200, 200), (320, 192), (400, 200)]
# (K, output channels per convolution, E).  "limits": the ABI's maxima (forward with four 64-channel chunks, weight gradient with
# K + E = 136 > 128 columns); "narrow": N_out <= 64 (one chunk) and a folded K % 32 != 0, whose egopose rows lie inside the input
# tile's zero-filled rows
BLOCKS = {"first": (70, [35, 35, 35, 64], 0), "second": (64, [32, 32, 32], 0), "folded": (64, [35, 35, 35, 64], 6),
          "limits": (128, [64, 64, 64, 64], 8), "narrow": (40, [8, 27], 8)}
SHIPPED = ("first", "second", "folded")


@pytest.fixture(autouse=True, scope="module")
def _no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _nerr(a, b):
    return TO.normwise_error(a, b)


def _input(b, k, s, h, w, layout, gen, ints=True):
    """(b, k, s, h, w) as the first block sees it (frame-major: the permuted (b, s, k, h, w) concat) or as the second does
    (channel-major: a contiguous NCDHW tensor)."""
    shape = (b, s, k, h, w) if layout == "frame_major" else (b, k, s, h, w)
    t = torch.randint(-2, 3, shape, generator=gen).float() if ints else torch.randn(shape, generator=gen)
    t = t.to(DEV)
    return t.permute(0, 2, 1, 3, 4) if layout == "frame_major" else t


def _weights(k, e, segs, gen, ints=True):
    mk = (lambda c: torch.randint(-2, 3, (c, k + e, 1, 1, 1), generator=gen).float()) if ints else \
        (lambda c: torch.randn((c, k + e, 1, 1, 1), generator=gen) / (k + e) ** 0.5)
    return [mk(c).to(DEV) for c in segs]


def _reference(x, ws, extra, grads):
    """fp64: the concat of x and the broadcast extra, the four convs, and their gradients."""
    xd = x.double()
    if extra is not None:
        b, _, s, h, w = x.shape
        xd = torch.cat([xd, extra.double().permute(0, 2, 1)[..., None, None].expand(b, -1, s, h, w)], 1)
    xd = xd.detach().requires_grad_(True)
    wd = [w.double().detach().requires_grad_(True) for w in ws]
    ys = [F.conv3d(xd, w) for w in wd]
    torch.autograd.backward(ys, [g.double() for g in grads])
    k = x.shape[1]
    return ys, xd.grad[:, :k], [w.grad for w in wd]


def _case(name, grid, b, s, layout, seed, ints=True):
    k, segs, e = BLOCKS[name]
    gen = torch.Generator().manual_seed(seed)
    x = _input(b, k, s, *grid, layout, gen, ints)
    ws = _weights(k, e, segs, gen, ints)
    extra = None
    if e:
        extra = (torch.randint(-2, 3, (b, s, e), generator=gen).float() if ints else torch.randn((b, s, e), generator=gen)).to(DEV)
    grads = [(torch.randint(-2, 3, (b, c, s, *grid), generator=gen).float() if ints else torch.randn((b, c, s, *grid), generator=gen)).to(DEV)
             for c in segs]
    return x, ws, extra, grads


CASES = [(name, grid, bs, layout) for name in BLOCKS for grid in (GRIDS if name in SHIPPED else [(8, 8), (52, 49), (200, 200)])
         for bs, layout in (((1, 1), "channel_major"), ((3, 3), "frame_major"), ((1, 3), "frame_major"), ((3, 1), "channel_major"))]


@pytest.mark.parametrize("name,grid,bs,layout", CASES, ids=lambda v: str(v).replace(" ", ""))
def test_small_integers_bit_exact(name, grid, bs, layout):
    """Forward, input gradient and weight gradient equal fp64 exactly; every output, the workspace and the input gradient start
    NaN-filled (deterministic mode fills uninitialised memory), so an element a kernel does not write shows up."""
    b, s = bs
    x, ws, extra, grads = _case(name, grid, b, s, layout, seed=CASES.index((name, grid, bs, layout)))
    ys_ref, gx_ref, gw_ref = _reference(x, ws, extra, grads)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        ys = entry_forward(x, ws, extra)
        gx = entry_backward_data(grads, x, ws)
        gw = entry_backward_weight(grads, x, ws, extra)
    finally:
        torch.use_deterministic_algorithms(old)
    for y, r in zip(ys, ys_ref):
        assert y.is_contiguous() and torch.equal(y.double(), r)
    assert gx.stride() == x.stride() and torch.equal(gx.double(), gx_ref)
    for g, r in zip(gw, gw_ref):
        assert torch.equal(g.double(), r)


@pytest.mark.parametrize("name", list(BLOCKS))
@pytest.mark.parametrize("grid", [(52, 49), (200, 200)])
def test_random_fp32_against_fp64_and_cudnn(name, grid):
    x, ws, extra, grads = _case(name, grid, 3, 3, "frame_major" if name == "first" else "channel_major", seed=7, ints=False)
    ys_ref, gx_ref, gw_ref = _reference(x, ws, extra, grads)
    ys = entry_forward(x, ws, extra)
    gx = entry_backward_data(grads, x, ws)
    gw = entry_backward_weight(grads, x, ws, extra)
    # cuDNN TF32 on the concat, and fp64 on TF32-rounded operands
    torch.backends.cudnn.allow_tf32 = True
    try:
        ys_tf, gx_tf, gw_tf = _reference_f32(x, ws, extra, grads)
    finally:
        torch.backends.cudnn.allow_tf32 = False
    rnd = lambda t: _tf32(t)
    ys_r, gx_r, gw_r = _reference(rnd(x), [rnd(w) for w in ws], None if extra is None else rnd(extra), [rnd(g) for g in grads])
    got = (torch.cat([y.flatten() for y in ys]), gx, torch.cat([g.flatten() for g in gw]))
    ref = (torch.cat([y.flatten() for y in ys_ref]), gx_ref, torch.cat([g.flatten() for g in gw_ref]))
    tf = (torch.cat([y.flatten() for y in ys_tf]), gx_tf, torch.cat([g.flatten() for g in gw_tf]))
    rr = (torch.cat([y.flatten() for y in ys_r]), gx_r, torch.cat([g.flatten() for g in gw_r]))
    for what, g_, r_, t_, q_ in zip(("forward", "grad_x", "grad_w"), got, ref, tf, rr):
        err = _nerr(g_, r_)
        bar = 3 * max(_nerr(t_, r_), _nerr(q_, r_))
        assert err < 1e-3 and err <= bar, f"{what}: {err:.3e} (bar {bar:.3e})"


def _tf32(t):
    """round to TF32 (nearest, ties away), as cvt.rna does"""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).view(t.shape)


def _reference_f32(x, ws, extra, grads):
    xf = x.float()
    if extra is not None:
        b, _, s, h, w = x.shape
        xf = torch.cat([xf, extra.permute(0, 2, 1)[..., None, None].expand(b, -1, s, h, w)], 1)
    xf = xf.detach().requires_grad_(True)
    wf = [w.detach().clone().requires_grad_(True) for w in ws]
    ys = [F.conv3d(xf, w) for w in wf]
    torch.autograd.backward(ys, grads)
    return ys, xf.grad[:, :x.shape[1]], [w.grad for w in wf]


def test_reproducible_eager_and_graph_replay():
    x, ws, extra, grads = _case("folded", (200, 200), 3, 3, "frame_major", seed=3, ints=False)
    first = (entry_forward(x, ws, extra), entry_backward_data(grads, x, ws), entry_backward_weight(grads, x, ws, extra))
    for _ in range(2):
        again = (entry_forward(x, ws, extra), entry_backward_data(grads, x, ws), entry_backward_weight(grads, x, ws, extra))
        assert all(torch.equal(a, b) for a, b in zip(first[0] + [first[1]] + first[2], again[0] + [again[1]] + again[2]))
    entry_forward(x, ws, extra)                               # packs cached before capture
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        entry_forward(x, ws, extra)
        entry_backward_weight(grads, x, ws, extra)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ys = entry_forward(x, ws, extra)
        gx = entry_backward_data(grads, x, ws)
        gw = entry_backward_weight(grads, x, ws, extra)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(first[0] + [first[1]] + first[2], ys + [gx] + gw))


def test_zero_frames():
    x, ws, extra, grads = _case("folded", (8, 8), 1, 1, "channel_major", seed=1)
    x0 = x[:0]
    assert [tuple(y.shape) for y in entry_forward(x0, ws, extra[:0])] == [(0, c, 1, 8, 8) for c in (35, 35, 35, 64)]
    gw = entry_backward_weight([g[:0] for g in grads], x0, ws, extra[:0])
    assert all(torch.count_nonzero(g) == 0 for g in gw)


# ------------------------------------------------------------------------------------------------------------------------------
# modules
# ------------------------------------------------------------------------------------------------------------------------------
def _model(grid, rf=3, seed=0):
    torch.manual_seed(seed)
    m = TO.TemporalModel(70, rf, grid, start_out_channels=64)
    for mod in m.modules():                                   # non-trivial BN affine / running statistics
        if isinstance(mod, torch.nn.BatchNorm3d):
            mod.weight.data.uniform_(0.5, 1.5)
            mod.bias.data.uniform_(-0.2, 0.2)
            mod.running_mean.uniform_(-0.1, 0.1)
            mod.running_var.uniform_(0.5, 1.5)
    return m.to(DEV)


def _swapped(m):
    s = copy.deepcopy(m)
    install.use_tensor_core_temporal_model(type("M", (), {"temporal_model": s})())
    assert all(isinstance(b, TensorCoreTemporalBlock) for b in s.model)
    return s


def _run(m, x, gout, amp=False, tf32=False):
    """outputs, input gradient and parameter gradients of one step; tf32: cuDNN may use TF32 (the oracle's bar)"""
    x = x.detach().clone().requires_grad_(True)
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            y = m(x)
        y.float().backward(gout)
    finally:
        torch.backends.cudnn.allow_tf32 = False
    return y.float().detach(), x.grad, {n.replace("_orig_mod.", ""): p.grad.detach().clone() for n, p in m.named_parameters()}


@pytest.mark.parametrize("amp", [False, True], ids=["fp32", "amp"])
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
def test_whole_model_matches_oracle(train, amp):
    """Against fp64, within 3x of the oracle's own error with cuDNN in TF32 (fp32) or under the same autocast (amp).  In train mode
    BatchNorm's backward removes each channel's mean gradient, so the input gradient is a small difference of large terms: operand
    rounding shows up in it ~100x amplified, for cuDNN TF32 as for the kernels."""
    grid = (52, 48)
    ref = _model(grid)
    sw = _swapped(ref)
    ref64 = copy.deepcopy(ref).double()
    for m in (ref, sw, ref64):
        m.train(train)
    gen = torch.Generator().manual_seed(11)
    x = torch.randn((2, 3, 70, *grid), generator=gen).to(DEV)
    gout = torch.randn((2, 1, 64, *grid), generator=gen).to(DEV)
    y64, gx64, gp64 = _run(ref64, x.double(), gout.double())
    y0, gx0, gp0 = _run(ref, x, gout, amp, tf32=True)
    y1, gx1, gp1 = _run(sw, x, gout, amp)
    assert set(gp1) == set(gp0) == set(gp64)
    for what, a, r, o in [("out", y1, y64, y0), ("grad_x", gx1, gx64, gx0)] + [(n, gp1[n], gp64[n], gp0[n]) for n in gp64]:
        err, bar = _nerr(a, r), max(3 * _nerr(o, r), 1e-5)
        assert err <= bar, f"{what}: {err:.3e} vs oracle {_nerr(o, r):.3e}"
    if train:                                                   # running statistics follow the same batches
        for (n, b1), (_, b0) in zip(sw.named_buffers(), ref.named_buffers()):
            if b1.dtype.is_floating_point:
                assert _nerr(b1, b0) < 1e-3, n


def test_folded_route_matches_concat_route():
    grid = (52, 48)
    ref = _model(grid, seed=2)
    sw = _swapped(ref)
    sw.train(True)
    gen = torch.Generator().manual_seed(5)
    bev = torch.randn((2, 3, 64, *grid), generator=gen).to(DEV)
    ego = torch.randn((2, 3, 6), generator=gen).to(DEV)
    gout = torch.randn((2, 1, 64, *grid), generator=gen).to(DEV)
    ref64 = copy.deepcopy(ref).double().train(True)
    b64 = bev.double().requires_grad_(True)
    y64 = ref64(TO.egopose_concat(b64, ego.double()))
    y64.backward(gout.double())
    folded = copy.deepcopy(sw)
    bf = bev.clone().requires_grad_(True)
    yf = temporal_model_forward(folded, bf, ego)
    yf.backward(gout)
    bc = bev.clone().requires_grad_(True)
    yc = sw(TO.egopose_concat(bc, ego))
    yc.backward(gout)
    tf = copy.deepcopy(ref).train(True)                   # the bar: the oracle on the concat with cuDNN in TF32
    bt = bev.clone().requires_grad_(True)
    torch.backends.cudnn.allow_tf32 = True
    try:
        yt = tf(TO.egopose_concat(bt, ego))
        yt.backward(gout)
    finally:
        torch.backends.cudnn.allow_tf32 = False
    assert _nerr(yf, y64) < 1e-3
    for what, f, c, t, r in (("out", yf, yc, yt, y64), ("grad_bev", bf.grad, bc.grad, bt.grad, b64.grad)):
        bar = max(3 * _nerr(t, r), 1e-5)
        assert _nerr(f, r) <= bar and _nerr(c, r) <= bar, f"{what}: folded {_nerr(f, r):.3e} concat {_nerr(c, r):.3e} bar {bar:.3e}"
    gp64, gpt, gpc = dict(ref64.named_parameters()), dict(tf.named_parameters()), dict(sw.named_parameters())
    for n, pf in folded.named_parameters():
        r = gp64[n].grad
        bar = max(3 * _nerr(gpt[n].grad, r), 1e-5)
        assert _nerr(pf.grad, r) <= bar and _nerr(gpc[n].grad, r) <= bar, n


def test_full_chain_lift_warp_temporal():
    """forward_warped (lift + cumulative warp) -> folded temporal model, against the fp64 oracle chain on the same BEV."""
    from fiery_b200.lift import LiftSplat
    from fiery_b200.synthetic import CONFIGS, make_calibration, make_egomotion, make_head
    from oracle import lift_oracle as O
    from oracle import warp_oracle as W
    from fiery_b200.synthetic import LiftConfig
    s = 3
    cfg = LiftConfig(**{**CONFIGS["cfg1_tiny"].__dict__, "frames": s})       # one sequence of three frames
    calib = [torch.from_numpy(a) for a in make_calibration(cfg, seed=1)]
    head = torch.from_numpy(make_head(cfg, seed=1))
    flow = torch.from_numpy(make_egomotion(1, s, seed=0))
    ext = (float(cfg.x_bound[1]), float(cfg.y_bound[1]))
    lift = LiftSplat.from_config(cfg).to(DEV)
    bev = lift.forward_warped(head.to(DEV), calib[0].to(DEV), calib[1].to(DEV), flow.to(DEV), ext)     # (b, s, 64, X, Y)
    exact = O.LiftOracle.from_config(cfg).lift_exact(head, *calib)
    warped = W.cumulative_warp_features(exact.float().unflatten(0, (1, s)).clone(), flow, mode="bilinear", spatial_extent=ext)
    grid = tuple(bev.shape[-2:])
    if (grid[0] * grid[1]) % 4:
        pytest.skip("grid not covered")
    ref = _model(grid, rf=s, seed=4).eval()
    sw = _swapped(ref).eval()
    with torch.no_grad():
        got = temporal_model_forward(sw, bev, flow.to(DEV))
        want = copy.deepcopy(ref).double()(TO.egopose_concat(warped.double().to(DEV), flow.double().to(DEV)))
    assert _nerr(got, want) < 1e-3


# ------------------------------------------------------------------------------------------------------------------------------
# operators under the compiler
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["first", "folded"])
def test_opcheck(name):
    x, ws, extra, grads = _case(name, (8, 8), 2, 3, "frame_major", seed=9, ints=False)
    x = x.requires_grad_(True)
    ws = [w.requires_grad_(True) for w in ws]
    torch.library.opcheck(torch.ops.fiery_b200.temporal_entry.default, (x, ws, extra))
    for ni, nw in ((True, True), (True, False), (False, True)):
        torch.library.opcheck(torch.ops.fiery_b200.temporal_entry_backward.default, (grads, x.detach(), [w.detach() for w in ws], extra, ni, nw))


@pytest.mark.parametrize("backend", ["aot_eager", "inductor"])
def test_compiled_block_matches_eager(backend):
    grid = (52, 48)
    ref = _model(grid, seed=6)
    sw = _swapped(ref).train(True)
    comp = copy.deepcopy(sw)
    gen = torch.Generator().manual_seed(8)
    x = torch.randn((2, 3, 70, *grid), generator=gen).to(DEV)
    gout = torch.randn((2, 1, 64, *grid), generator=gen).to(DEV)
    ref64 = copy.deepcopy(ref).double().train(True)
    y64, gx64, gp64 = _run(ref64, x.double(), gout.double())
    y0, gx0, gp0 = _run(sw, x, gout)
    fn = torch.compile(comp, backend=backend, fullgraph=True)
    y1, gx1, gp1 = _run(fn, x, gout)
    assert set(gp1) == set(gp0)
    for what, a, e, r in [("out", y1, y0, y64), ("grad_x", gx1, gx0, gx64)] + [(n, gp1[n], gp0[n], gp64[n]) for n in gp0]:
        assert _nerr(a, r) <= max(1.5 * _nerr(e, r), 1e-5), f"{what}: compiled {_nerr(a, r):.3e} eager {_nerr(e, r):.3e}"


def test_frozen_weights_launch_no_weight_gradient(monkeypatch):
    """needs_input_grad decides which gradients run: frozen weights launch no weight gradient, a frozen input no input gradient."""
    from fiery_b200 import temporal
    calls = []
    for name in ("entry_backward_data", "entry_backward_weight"):
        monkeypatch.setattr(temporal, name, (lambda f, n: lambda *a, **k: calls.append(n) or f(*a, **k))(getattr(temporal, name), name))
    x, ws, extra, grads = _case("first", (8, 8), 1, 3, "frame_major", seed=2, ints=False)
    for need_x, need_w, want in ((True, False, ["entry_backward_data"]), (False, True, ["entry_backward_weight"]),
                                 (True, True, ["entry_backward_data", "entry_backward_weight"])):
        calls.clear()
        xi = x.detach().requires_grad_(need_x)
        wi = [w.detach().requires_grad_(need_w) for w in ws]
        torch.autograd.backward(torch.ops.fiery_b200.temporal_entry(xi, wi, None), grads)
        assert calls == want
        assert (xi.grad is not None) == need_x and all((w.grad is not None) == need_w for w in wi)
