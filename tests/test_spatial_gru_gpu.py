"""The SpatialGRU on the kernels (torch.ops.fiery_b200.spatial_gru, fiery_b200/future_prediction.py) against an fp64 copy of the
oracle module: outputs, every gradient and the running statistics, across the accepted channel splits, grids, batches and step
counts, train and eval, fp32 and autocast; bit-reproducibility; opcheck; graph replay; the swap of a whole FuturePrediction."""
from __future__ import annotations

import copy

import pytest
import torch
import torch.nn as nn

from oracle.future_oracle import FuturePrediction, SpatialGRU

pytestmark = pytest.mark.gpu


def _randomize(m: nn.Module, seed: int) -> nn.Module:
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (0.5 if p.dim() == 1 else 0.2) / (1 if p.dim() == 1 else p.shape[1] ** 0.5 / 2))
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.weight.add_(1.0)
                mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
    return m


def _swap(m: nn.Module) -> nn.Module:
    from fiery_b200.future_prediction import TensorCoreSpatialGRU
    return TensorCoreSpatialGRU.from_module(m)


def _rel(a: torch.Tensor, ref: torch.Tensor) -> float:
    return float((a.detach().double() - ref.detach().double()).norm() / ref.detach().double().norm().clamp_min(1e-30))


# The bar: 3x the reference module's own fp32 CUDA error against fp64, and never below 1e-3 normwise, the TF32 operand rounding
# (2^-11 relative per operand) the kernels take by design: where cuDNN picks an exact fp32 algorithm (small widths) its error is far
# below TF32's.
TF32_FLOOR = 1e-3


def _within(e: float, e_ref: float) -> bool:
    return e <= max(3 * e_ref, TF32_FLOOR)


def _tf32(t: torch.Tensor) -> torch.Tensor:
    """t with its values rounded to TF32 (10 mantissa bits, ties away from zero, as cvt.rna), gradient passed straight through"""
    bits = t.detach().float().contiguous().view(torch.int32)
    r = ((bits + 0x1000) & ~0x1FFF).view(torch.float32).to(t.dtype)
    return t + (r - t).detach()


def _tf32_operands(m: nn.Module) -> nn.Module:
    """m (an fp64 copy) with every Conv2d's input and weight rounded to TF32 first: the operand rounding the kernels do, without their
    accumulation order -- what "fp64 on TF32-rounded operands" means for a whole module"""
    for conv in m.modules():
        if isinstance(conv, nn.Conv2d):
            conv.forward = (lambda c: lambda x: torch.nn.functional.conv2d(_tf32(x), _tf32(c.weight), c.bias, c.stride, c.padding))(conv)
    return m


def _run(module, x, h0, gout):
    x = x.clone().requires_grad_(True)
    h0 = h0.clone().requires_grad_(True)
    out = module(x, h0)
    out.backward(gout)
    grads = {"x": x.grad, "h0": h0.grad}
    grads.update({n: p.grad for n, p in module.named_parameters()})
    return out.detach(), grads


def _inputs(b, T, cx, ch, h, w, broadcast, seed, dev="cuda"):
    g = torch.Generator().manual_seed(seed)
    if broadcast:
        x = torch.randn(b, 1, cx, 1, 1, generator=g).expand(b, T, cx, h, w)
    else:
        x = torch.randn(b, T, cx, h, w, generator=g)
    h0 = torch.randn(b, ch, h, w, generator=g)
    gout = torch.randn(b, T, ch, h, w, generator=g)
    return x.to(dev), h0.to(dev), gout.to(dev)


CASES = [
    # cx, ch, h, w, b, T, broadcast x, gru_bias_init
    (32, 64, 12, 16, 2, 4, True, 0.0),
    (64, 64, 7, 12, 1, 5, False, 0.0),
    (1, 8, 1, 4, 3, 1, False, 0.0),
    (35, 29, 9, 20, 2, 4, False, 0.0),
    (64, 1, 10, 8, 1, 4, False, 0.0),
    (32, 64, 40, 24, 3, 4, False, 0.0),
    (32, 48, 12, 16, 2, 4, True, 0.0),          # C_h in 33..60: the gates' weight gradient has a 32-channel second block
    (64, 40, 9, 20, 2, 5, False, 0.0),
    (16, 24, 8, 12, 2, 3, False, 0.75),         # a non-zero gru_bias_init
]


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "cx{}_ch{}_{}x{}_b{}_T{}{}{}".format(*c[:6], "_bcast" if c[6] else "",
                                                                                       f"_g{c[7]}" if c[7] else ""))
def test_against_fp64(case, training):
    cx, ch, h, w, b, T, broadcast, bias_init = case
    base = _randomize(SpatialGRU(cx, ch, gru_bias_init=bias_init), 1 + cx + ch).cuda().train(training)
    ref64 = copy.deepcopy(base).double()
    ref32 = copy.deepcopy(base)
    ours = _swap(copy.deepcopy(base))
    x, h0, gout = _inputs(b, T, cx, ch, h, w, broadcast, 7)
    o64, g64 = _run(ref64, x.double(), h0.double(), gout.double())
    o32, g32 = _run(ref32, x, h0, gout)
    ot, gt = _run(_tf32_operands(copy.deepcopy(base).double()), x.double(), h0.double(), gout.double())
    o, g = _run(ours, x, h0, gout)
    assert o.dtype == torch.float32 and o.shape == (b, T, ch, h, w)
    # the reference error: the larger of torch's fp32 CUDA module (cuDNN TF32, or exact fp32 where cuDNN picks it) and fp64 on
    # TF32-rounded operands
    errs = {"out": (_rel(o, o64), max(_rel(o32, o64), _rel(ot, o64)))}
    for k in g64:
        errs[k] = (_rel(g[k], g64[k]), max(_rel(g32[k], g64[k]), _rel(gt[k], g64[k])))
    for k, (e, e_ref) in errs.items():
        assert _within(e, e_ref), (k, e, e_ref, errs)
    bn, bn64 = ours.conv_state_tilde.norm, ref64.conv_state_tilde.norm
    assert int(bn.num_batches_tracked) == int(bn64.num_batches_tracked) == (T if training else 0)
    assert _rel(bn.running_mean, bn64.running_mean) < 1e-3
    assert _rel(bn.running_var, bn64.running_var) < 1e-3


def test_large_grid_ragged_tiles():
    # 200 x 200 (and a 400-row map) at the project's widths: ragged 8 x 16 tiles on both edges
    for (h, w, cx) in ((200, 200, 32), (400, 200, 64)):
        base = _randomize(SpatialGRU(cx, 64), 5).cuda()
        ref64, ref32 = copy.deepcopy(base).double(), copy.deepcopy(base)
        ours = _swap(copy.deepcopy(base))
        x, h0, gout = _inputs(1, 2, cx, 64, h, w, False, 3)
        o64, g64 = _run(ref64, x.double(), h0.double(), gout.double())
        o32, g32 = _run(ref32, x, h0, gout)
        o, g = _run(ours, x, h0, gout)
        assert _within(_rel(o, o64), _rel(o32, o64))
        for k in g64:
            assert _within(_rel(g[k], g64[k]), _rel(g32[k], g64[k])), k


def test_autocast_and_momentum_none():
    base = _randomize(SpatialGRU(32, 64), 11).cuda()
    base.conv_state_tilde.norm.momentum = None
    ref64 = copy.deepcopy(base).double()
    ours = _swap(copy.deepcopy(base))
    x, h0, gout = _inputs(2, 4, 32, 64, 12, 16, True, 9)
    o64, g64 = _run(ref64, x.double(), h0.double(), gout.double())
    with torch.autocast("cuda", dtype=torch.float16):
        xo = x.clone().requires_grad_(True)
        out = ours(xo, h0)
    assert out.dtype == torch.float32
    out.backward(gout)
    ref32 = copy.deepcopy(base)
    o32, g32 = _run(ref32, x, h0, gout)
    assert _within(_rel(out, o64), _rel(o32, o64))
    assert _within(_rel(xo.grad, g64["x"]), _rel(g32["x"], g64["x"]))
    bn, bn64 = ours.conv_state_tilde.norm, ref64.conv_state_tilde.norm
    assert _rel(bn.running_var, bn64.running_var) < 1e-3 and int(bn.num_batches_tracked) == 4


def test_bit_reproducible_and_independent_of_buffer_contents(monkeypatch):
    base = _randomize(SpatialGRU(64, 64), 2).cuda()
    ours = _swap(base)
    x, h0, gout = _inputs(2, 4, 64, 64, 24, 20, False, 4)
    o1, g1 = _run(ours, x, h0, gout)
    for p in ours.parameters():
        p.grad = None
    # every buffer the operator allocates -- outputs, saved tensors, gradients, workspaces -- starts full of NaN bits
    empty = torch.empty

    def nan_empty(*args, **kwargs):
        t = empty(*args, **kwargs)
        if t.is_cuda:
            (t.fill_(255) if t.dtype == torch.uint8 else t.fill_(float("nan")) if t.is_floating_point() else t)
        return t

    monkeypatch.setattr(torch, "empty", nan_empty)
    o2, g2 = _run(ours, x, h0, gout)
    monkeypatch.undo()
    assert torch.equal(o1, o2)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k


def test_gradient_subsets():
    base = _randomize(SpatialGRU(16, 24), 3).cuda()
    ours = _swap(base)
    x, h0, gout = _inputs(1, 3, 16, 24, 8, 8, False, 5)
    full_o, full_g = _run(ours, x, h0, gout)
    for p in ours.parameters():
        p.requires_grad_(False)
        p.grad = None
    xo = x.clone().requires_grad_(True)
    ours(xo, h0).backward(gout)
    assert torch.equal(xo.grad, full_g["x"])
    for p in ours.parameters():
        p.requires_grad_(True)


def test_graph_replay():
    # eval forward, and a training forward + backward with its running-statistics updates
    base = _randomize(SpatialGRU(32, 64), 8).cuda().eval()
    ours = _swap(base)
    x, h0, gout = _inputs(2, 4, 32, 64, 16, 16, False, 6)
    eager = ours(x, h0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ours(x, h0)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ours(x, h0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)

    train = _randomize(SpatialGRU(32, 64), 9).cuda().train()
    eager_m, graph_m = _swap(copy.deepcopy(train)), _swap(copy.deepcopy(train))
    xg, hg = x.clone().requires_grad_(True), h0.clone().requires_grad_(True)

    def step(m, xx, hh):
        y = m(xx, hh)
        y.backward(gout)
        return y

    for _ in range(2):                                   # two eager steps: the reference for two replays
        xe, he = x.clone().requires_grad_(True), h0.clone().requires_grad_(True)
        ye = step(eager_m, xe, he)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(graph_m, xg, hg)                            # warm-up: one update of the running statistics
    torch.cuda.current_stream().wait_stream(s)
    for p in list(graph_m.parameters()) + [xg, hg]:
        p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg = step(graph_m, xg, hg)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg.detach(), ye.detach())
    assert torch.equal(xg.grad, xe.grad) and torch.equal(hg.grad, he.grad)
    bn_e, bn_g = eager_m.conv_state_tilde.norm, graph_m.conv_state_tilde.norm
    assert torch.equal(bn_g.running_mean, bn_e.running_mean) and torch.equal(bn_g.running_var, bn_e.running_var)
    assert int(bn_g.num_batches_tracked) == int(bn_e.num_batches_tracked) == 8


def test_opcheck():
    base = _randomize(SpatialGRU(8, 16), 4).cuda()
    x, h0, _ = _inputs(1, 2, 8, 16, 4, 8, False, 2)
    bn = base.conv_state_tilde.norm
    args = (x.requires_grad_(True), h0.requires_grad_(True), base.conv_update.weight, base.conv_update.bias, base.conv_reset.weight,
            base.conv_reset.bias, base.conv_state_tilde.conv.weight, bn.weight, bn.bias, None, None, 2, True, bn.eps, 0.0)
    import fiery_b200.future_prediction  # noqa: F401
    torch.library.opcheck(torch.ops.fiery_b200.spatial_gru.default, args,
                          test_utils=("test_schema", "test_faketensor", "test_autograd_registration"))


def test_whole_future_prediction_swapped():
    from fiery_b200.install import use_tensor_core_future_prediction

    class Holder(nn.Module):
        def __init__(self, fp):
            super().__init__()
            self.future_prediction = fp

    fp = _randomize(FuturePrediction(64, 32), 12).cuda()
    ref64 = copy.deepcopy(fp).double()
    ref32 = copy.deepcopy(fp)
    model = Holder(copy.deepcopy(fp))
    keys = list(model.state_dict().keys())
    use_tensor_core_future_prediction(model)
    use_tensor_core_future_prediction(model)
    assert list(model.state_dict().keys()) == keys
    g = torch.Generator().manual_seed(1)
    b, T, h, w = 2, 4, 16, 20
    x = (torch.randn(b, 1, 32, 1, 1, generator=g)).expand(b, T, 32, h, w).cuda()
    h0 = torch.randn(b, 64, h, w, generator=g).cuda()
    gout = torch.randn(b, T, 64, h, w, generator=g).cuda()

    def run(m, dtype):
        hh = h0.to(dtype).requires_grad_(True)
        out = m(x.to(dtype), hh)
        out.backward(gout.to(dtype))
        return out.detach(), hh.grad, {n: p.grad for n, p in m.named_parameters()}

    o64, h64, p64 = run(ref64, torch.float64)
    o32, h32, p32 = run(ref32, torch.float32)
    o, hg, pg = run(model.future_prediction, torch.float32)
    assert _within(_rel(o, o64), _rel(o32, o64))
    assert _within(_rel(hg, h64), _rel(h32, h64))
    for n in p64:
        assert _within(_rel(pg[n], p64[n]), _rel(p32[n], p64[n])), n


def test_no_map_ops_inside_the_swapped_gru():
    base = _randomize(SpatialGRU(32, 64), 13).cuda()
    ours = _swap(base)
    x, h0, gout = _inputs(2, 4, 32, 64, 16, 16, True, 3)
    _run(ours, x, h0, gout)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU], acc_events=True) as prof:
        _run(ours, x, h0, gout)
    names = {e.name for e in prof.events()}
    banned = [n for n in names if n in ("aten::cat", "aten::sigmoid", "aten::convolution", "aten::cudnn_convolution",
                                        "aten::batch_norm", "aten::cudnn_batch_norm", "aten::stack")]
    assert not banned, banned


def test_torch_compile_matches_eager():
    base = _randomize(SpatialGRU(32, 64), 14).cuda()
    eager_m, comp_m = _swap(copy.deepcopy(base)), _swap(copy.deepcopy(base))
    x, h0, gout = _inputs(2, 3, 32, 64, 8, 12, False, 8)
    o1, g1 = _run(eager_m, x, h0, gout)
    compiled = torch.compile(comp_m, backend="aot_eager", fullgraph=False)
    xo, ho = x.clone().requires_grad_(True), h0.clone().requires_grad_(True)
    out = compiled(xo, ho)
    out.backward(gout)
    assert torch.equal(out.detach(), o1)
    assert torch.equal(xo.grad, g1["x"]) and torch.equal(ho.grad, g1["h0"])
    for n, p in comp_m.named_parameters():
        assert torch.equal(p.grad, g1[n]), n
    assert torch.equal(comp_m.conv_state_tilde.norm.running_mean, eager_m.conv_state_tilde.norm.running_mean)
