"""GPU: the temporal block's pyramid pooling and aggregation on the kernels -- the spatial sums (csrc/spatial_sums.cu) and
``temporal_aggregation`` (the entry's kernels in swapped roles, csrc/temporal_entry.cu) against fp64, their reproducibility, the
operators under opcheck and the compiler, and whole TemporalModels with the pyramid-pooling swap against the fp64 oracle
(oracle/temporal_oracle.py), with the ops a swapped step dispatches.

Parity bars as tests/test_temporal_entry_gpu.py: small integers are exact in TF32 and fp32, so on them every output and gradient
is bit-exact; random fp32 within 3x of the larger of cuDNN TF32's error and fp64 on TF32-rounded operands; whole models within 3x
of the oracle's own error (cuDNN in TF32 for fp32, the same autocast for AMP)."""
import copy

import pytest
import torch
import torch.nn.functional as F
from torch.utils._python_dispatch import TorchDispatchMode

from fiery_b200 import _lib, install, ops  # noqa: F401  (registers the operators)
from fiery_b200.temporal import TensorCorePyramidPooling, TensorCoreTemporalBlock, aggregation_backward, aggregation_forward, \
    spatial_sums, temporal_model_forward
from oracle import temporal_oracle as TO
from tests._temporal_models import temporal_model

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True, scope="module")
def _no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _nerr(a, b):
    return TO.normwise_error(a, b)


def _tf32(t):
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).view(t.shape)


# ------------------------------------------------------------------------------------------------------------------------------
# spatial sums
# ------------------------------------------------------------------------------------------------------------------------------
# pixel counts around the kernel's loop edges too: 1024 pixels are one pass of 256 threads over 4-pixel chunks, 4096 one unrolled pass
SUM_GRIDS = [(1, 1), (1, 3), (3, 5), (8, 8), (52, 49), (200, 200), (400, 200),
             (3, 341), (32, 32), (5, 205), (3, 1365), (64, 64), (17, 241), (3, 2731)]


def _sums_guarded(x):
    """the C entry point into a NaN-guarded buffer: (sums, guards intact)"""
    b, c, s, h, w = x.shape
    n = b * c * s
    buf = torch.full((n + 64,), float("nan"), device=DEV)
    d = _lib.SpatialSumsDesc()
    d.batch, d.channels, d.frames, d.pixels = b, c, s, h * w
    d.stride_b, d.stride_c, d.stride_t = x.stride(0), x.stride(1), x.stride(2)
    _lib.call("fiery_spatial_sums", DEV, d, x.data_ptr(), buf[32:].data_ptr())
    torch.cuda.synchronize()
    return buf[32:32 + n].view(b, c, s), bool(torch.isnan(buf[:32]).all() and torch.isnan(buf[32 + n:]).all())


@pytest.mark.parametrize("grid", SUM_GRIDS, ids=str)
@pytest.mark.parametrize("frames", [0, 1, 3])
def test_sums_small_integers_bit_exact_every_layout(grid, frames):
    gen = torch.Generator().manual_seed(grid[0] * 1000 + grid[1] + frames)
    base = torch.randint(-3, 4, (2, frames, 20, *grid), generator=gen).float().to(DEV)       # (b, s, C, X, Y)
    permuted = base.permute(0, 2, 1, 3, 4)                                                    # (b, C, s, X, Y) frame-major
    contiguous = permuted.contiguous()
    sliced = contiguous[:, 3:17]                                                              # a channel slice
    want = permuted.double().sum(dim=(3, 4))
    results = []
    for x in (permuted, contiguous, sliced):
        got, guards = _sums_guarded(x)
        assert guards
        results.append(got)
        ref = want if x is not sliced else want[:, 3:17]
        assert torch.equal(got.double(), ref)
    assert torch.equal(results[0], results[1]) and torch.equal(results[0][:, 3:17], results[2])


@pytest.mark.parametrize("grid", [(3, 5), (52, 49), (200, 200), (400, 200)], ids=str)
def test_sums_random_fp32_and_plane_position(grid):
    gen = torch.Generator().manual_seed(1)
    x = torch.randn((3, 3, 64, *grid), generator=gen).to(DEV).permute(0, 2, 1, 3, 4)
    got = spatial_sums(x)
    ref = x.double().sum(dim=(3, 4))
    assert _nerr(got, ref) < 1e-6
    # the same plane alone, at another address (not 16-byte aligned), gives the same bits
    flat = torch.empty(grid[0] * grid[1] + 1, device=DEV)
    flat[1:] = x[1, 5, 2].flatten()
    one = flat[1:].view(1, 1, 1, *grid)
    assert torch.equal(spatial_sums(one).flatten(), got[1, 5, 2].flatten())


def test_sums_operator_gradient_is_the_broadcast():
    x = torch.randn(2, 5, 3, 6, 8, device=DEV, requires_grad=True)
    g = torch.randn(2, 5, 3, device=DEV)
    torch.ops.fiery_b200.spatial_sums(x).backward(g)
    assert torch.equal(x.grad, g[..., None, None].expand(x.shape))
    torch.library.opcheck(torch.ops.fiery_b200.spatial_sums.default, (x,))


# ------------------------------------------------------------------------------------------------------------------------------
# temporal_aggregation
# ------------------------------------------------------------------------------------------------------------------------------
# (path channels, R, N)
AGG = {"first": ((35, 35, 35), 23, 64), "second": ((32, 32, 32), 21, 64), "narrow": ((1, 8, 8), 1, 8)}


def _agg_case(name, grid, b, s, seed, ints=True):
    segs, r, n = AGG[name]
    gen = torch.Generator().manual_seed(seed)
    mk = (lambda *sh: torch.randint(-2, 3, sh, generator=gen).float()) if ints else (lambda *sh: torch.randn(sh, generator=gen))
    paths = [mk(b, c, s, *grid).to(DEV) for c in segs]
    weight = mk(n, sum(segs) + r, 1, 1, 1).to(DEV)
    if not ints:
        weight = weight / (sum(segs) + r) ** 0.5
    pooled = mk(b, r, s).to(DEV)
    grad = mk(b, n, s, *grid).to(DEV)
    return paths, weight, pooled, grad


def _agg_reference(paths, weight, pooled, grad, dtype=torch.float64):
    ps = [p.to(dtype).detach().requires_grad_(True) for p in paths]
    w = weight.to(dtype).detach().requires_grad_(True)
    v = pooled.to(dtype).detach().requires_grad_(True)
    b, _, s, h, wd = paths[0].shape
    z = F.conv3d(torch.cat(ps + [v[..., None, None].expand(*v.shape, h, wd)], 1), w)
    z.backward(grad.to(dtype))
    return z, [p.grad for p in ps], w.grad, v.grad


AGG_CASES = [(name, grid, bs) for name in AGG for grid in [(2, 2), (8, 8), (52, 48), (200, 200)] for bs in ((1, 1), (3, 3), (2, 3))]


@pytest.mark.parametrize("name,grid,bs", AGG_CASES, ids=lambda v: str(v).replace(" ", ""))
def test_aggregation_small_integers_bit_exact(name, grid, bs):
    """forward, path gradients, weight gradient (path and pooled columns) and pooled gradient equal fp64 exactly; outputs start
    NaN-filled (deterministic mode fills uninitialised memory)."""
    paths, weight, pooled, grad = _agg_case(name, grid, *bs, seed=AGG_CASES.index((name, grid, bs)))
    z_ref, gp_ref, gw_ref, gv_ref = _agg_reference(paths, weight, pooled, grad)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        z = aggregation_forward(paths, weight, pooled)
        gp, gw, gv = aggregation_backward(grad, paths, weight, pooled, True, True, True)
    finally:
        torch.use_deterministic_algorithms(old)
    assert z.is_contiguous() and torch.equal(z.double(), z_ref)
    for a, r in zip(gp, gp_ref):
        assert a.is_contiguous() and torch.equal(a.double(), r)
    assert torch.equal(gw.double(), gw_ref) and torch.equal(gv.double(), gv_ref)


@pytest.mark.parametrize("name", list(AGG))
def test_aggregation_random_fp32_against_fp64_and_cudnn(name):
    paths, weight, pooled, grad = _agg_case(name, (200, 200), 3, 3, seed=7, ints=False)
    ref = _agg_reference(paths, weight, pooled, grad)
    z = aggregation_forward(paths, weight, pooled)
    gp, gw, gv = aggregation_backward(grad, paths, weight, pooled, True, True, True)
    torch.backends.cudnn.allow_tf32 = True
    try:
        tf = _agg_reference(paths, weight, pooled, grad, torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32 = False
    rr = _agg_reference([_tf32(p) for p in paths], _tf32(weight), _tf32(pooled), _tf32(grad))
    flat = lambda o: (o[0], torch.cat([t.flatten() for t in o[1]]), o[2], o[3])
    for what, g_, r_, t_, q_ in zip(("forward", "grad_paths", "grad_weight", "grad_pooled"), flat((z, gp, gw, gv)), flat(ref),
                                     flat(tf), flat(rr)):
        err = _nerr(g_, r_)
        bar = max(3 * max(_nerr(t_, r_), _nerr(q_, r_)), 1e-6)
        assert err < 1e-3 and err <= bar, f"{what}: {err:.3e} (bar {bar:.3e})"


def test_aggregation_weight_gradient_reproducible_and_graph_replay():
    paths, weight, pooled, grad = _agg_case("first", (200, 200), 3, 3, seed=3, ints=False)
    first = aggregation_backward(grad, paths, weight, pooled, True, True, True)
    z0 = aggregation_forward(paths, weight, pooled)
    for _ in range(2):
        again = aggregation_backward(grad, paths, weight, pooled, True, True, True)
        assert torch.equal(again[1], first[1]) and torch.equal(again[2], first[2])
        assert all(torch.equal(a, b) for a, b in zip(again[0], first[0]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        aggregation_forward(paths, weight, pooled)
        aggregation_backward(grad, paths, weight, pooled, True, True, True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        z = aggregation_forward(paths, weight, pooled)
        out = aggregation_backward(grad, paths, weight, pooled, True, True, True)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(z, z0) and torch.equal(out[1], first[1]) and torch.equal(out[2], first[2])


def test_aggregation_opcheck():
    paths, weight, pooled, grad = _agg_case("first", (8, 8), 2, 3, seed=9, ints=False)
    paths = [p.requires_grad_(True) for p in paths]
    torch.library.opcheck(torch.ops.fiery_b200.temporal_aggregation.default, (paths, weight.requires_grad_(True), pooled.requires_grad_(True)))
    for need in ((True, True, True), (True, False, False), (False, True, False), (False, False, True)):
        torch.library.opcheck(torch.ops.fiery_b200.temporal_aggregation_backward.default,
                              (grad, [p.detach() for p in paths], weight.detach(), pooled.detach(), *need))


def test_frozen_weight_and_input_launch_only_what_is_asked(monkeypatch):
    calls = []
    real = _lib.call
    monkeypatch.setattr(_lib, "call", lambda entry, *a: calls.append(entry) or real(entry, *a))
    paths, weight, pooled, grad = _agg_case("second", (8, 8), 1, 3, seed=2, ints=False)
    for need_p, need_w, need_v, want in ((True, False, False, ["fiery_temporal_entry_forward"]),
                                         (False, True, False, ["fiery_spatial_sums", "fiery_temporal_entry_backward_weight"]),
                                         (False, False, True, ["fiery_spatial_sums"])):
        pi = [p.detach().requires_grad_(need_p) for p in paths]
        wi = weight.detach().requires_grad_(need_w)
        vi = pooled.detach().requires_grad_(need_v)
        z = torch.ops.fiery_b200.temporal_aggregation(pi, wi, vi)
        calls.clear()
        z.backward(grad)
        assert calls == want, (need_p, need_w, need_v, calls)
        assert all((p.grad is not None) == need_p for p in pi) and (wi.grad is not None) == need_w and (vi.grad is not None) == need_v


# ------------------------------------------------------------------------------------------------------------------------------
# whole TemporalModel
# ------------------------------------------------------------------------------------------------------------------------------
GRID = (52, 48)


def _model(rf, inbetween, seed=0, grid=GRID, start_out_channels=64, **kw):
    torch.manual_seed(seed)
    m = temporal_model(70, rf, grid, start_out_channels=start_out_channels, inbetween_layers=inbetween, **kw)
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
    blocks = [b for b in s.model if type(b).__name__ in ("TemporalBlock", "TensorCoreTemporalBlock")]
    assert all(isinstance(b.pyramid_pooling, TensorCorePyramidPooling) for b in blocks)
    assert all(isinstance(b, TensorCoreTemporalBlock) for b in blocks) == (swaps == "all")
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
               (("all", "concat"), ("all", "folded"), ("pool", "concat"))]


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
    if train:
        for (n, b1), (_, b0) in zip(sw.named_buffers(), ref.named_buffers()):
            if b1.dtype.is_floating_point:
                assert _nerr(b1, b0) < 1e-3, n


@pytest.mark.parametrize("backend", ["aot_eager", "inductor"])
def test_compiled_model_matches_eager(backend):
    ref = _model(3, 0, seed=6)
    sw = _swapped(ref, "all").train(True)
    comp = copy.deepcopy(sw)
    gen = torch.Generator().manual_seed(8)
    x = torch.randn((2, 3, 70, *GRID), generator=gen).to(DEV)
    gout = torch.randn((2, 1, 64, *GRID), generator=gen).to(DEV)

    def run(m):
        xi = x.clone().requires_grad_(True)
        y = m(xi)
        y.backward(gout)
        return y.detach(), xi.grad, {n.replace("_orig_mod.", ""): p.grad.detach().clone() for n, p in m.named_parameters()}

    ref64 = copy.deepcopy(ref).double().train(True)
    xi = x.double().requires_grad_(True)
    y64 = ref64(xi)
    y64.backward(gout.double())
    gx64, gp64 = xi.grad, {n: p.grad for n, p in ref64.named_parameters()}
    y0, gx0, gp0 = run(sw)
    y1, gx1, gp1 = run(torch.compile(comp, backend=backend, fullgraph=True))
    assert set(gp1) == set(gp0)
    for what, a, e, r in [("out", y1, y0, y64), ("grad_x", gx1, gx0, gx64)] + [(n, gp1[n], gp0[n], gp64[n]) for n in gp0]:
        assert _nerr(a, r) <= max(1.5 * _nerr(e, r), 1e-5), f"{what}: compiled {_nerr(a, r):.3e} eager {_nerr(e, r):.3e}"


class _Recorder(TorchDispatchMode):
    def __init__(self):
        super().__init__()
        self.ops = []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        self.ops.append((str(func.overloadpacket.__name__), args, out))
        return out


@pytest.mark.parametrize("route", ["concat", "folded"])
def test_swapped_step_dispatches_no_upsampling_pool_or_concat(route):
    ref = _model(3, 0, seed=1)
    sw = _swapped(ref, "all").train(True)
    gen = torch.Generator().manual_seed(2)
    bev = torch.randn((2, 3, 64, *GRID), generator=gen).to(DEV).requires_grad_(True)
    ego = torch.randn((2, 3, 6), generator=gen).to(DEV)
    agg_in = {b.aggregation[0].conv.in_channels for b in sw.model}
    with _Recorder() as rec:
        y = temporal_model_forward(sw, bev, ego) if route == "folded" else sw(TO.egopose_concat(bev, ego))
        y.sum().backward()
    names = [n for n, _, _ in rec.ops]
    assert not any(n.startswith("upsample_bilinear2d") for n in names)
    assert not any(n.startswith("avg_pool3d") for n in names)
    for n, _, out in rec.ops:
        if n == "cat" and isinstance(out, torch.Tensor) and out.dim() == 5:
            assert not (out.shape[1] in agg_in and tuple(out.shape[3:]) == GRID), "a concat feeds the aggregation"
    assert "temporal_aggregation" in names and "spatial_sums" in names
