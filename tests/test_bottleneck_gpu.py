"""The future prediction's Bottleneck on the kernels (fiery_bottleneck_*, torch.ops.fiery_b200.bottleneck, TensorCoreBottleneck).

1. Fused = unfused, bit for bit: every stage and gradient of the C ABI against the chain of today's entry points on the same inputs,
   written from NaN-filled memory between sentinel margins, over tile and halo edges, 1 and 12 maps, train and eval.
2. The padding belongs to relu(bn1(y1)): with scale 0 and shift 1 the normalized map is 1 inside and 0 outside.
3. The module against an fp64 copy of the oracle's Bottleneck, and a whole swapped FuturePrediction.
4. Reproducibility, graph replay, opcheck, torch.compile, gradient subsets, dispatch, memory and the fallbacks.
"""
from __future__ import annotations

import copy
import warnings

import pytest
import torch
import torch.nn as nn

from oracle.future_oracle import Bottleneck, FuturePrediction
from tests._bottleneck_cases import (GRAD_KEYS, SHAPES, SMALL, fused_backward, fused_forward, margins_intact, operands, unfused)

pytestmark = pytest.mark.gpu


def _ids(s):
    return "x".join(str(v) for v in s)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("shape", SHAPES, ids=_ids)
def test_fused_equals_unfused(shape, training):
    x, weights, norms = operands(*shape, seed=sum(shape))
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(7)).cuda()
    ref = unfused(x, weights, norms, training, g)
    (out, y1, y2, y3, stats), bufs = fused_forward(x, weights, norms, training)
    for name, got in (("y1", y1), ("y2", y2), ("y3", y3), ("out", out), ("stats", stats)):
        assert _bits_equal(got, ref[name]), name
    grads, gbufs = fused_backward(g, x, y1, y2, y3, stats, weights, norms, training)
    for name, got in zip(GRAD_KEYS, grads):
        assert _bits_equal(got, ref[name].view(got.shape)), name
    assert all(margins_intact(b) for b in bufs + gbufs)


@pytest.mark.parametrize("shape", SMALL, ids=_ids)
def test_padding_is_the_normalized_maps(shape):
    """bn1 and bn2 with weight 0 and bias 1: relu(bn(y)) is 1 at every map position, and must stay 0 in the 3x3 padding and past the
    1x1 tiles' last pixel.  Transforming the zero fill instead would put 1s there and change y2, y3 and the weight gradients."""
    x, weights, norms = operands(*shape, seed=3)
    for i in (0, 4):
        norms[i] = torch.zeros_like(norms[i])
        norms[i + 1] = torch.ones_like(norms[i + 1])
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(8)).cuda()
    ref = unfused(x, weights, norms, True, g)
    (out, y1, y2, y3, stats), _ = fused_forward(x, weights, norms, True)
    for name, got in (("y2", y2), ("y3", y3), ("out", out)):
        assert _bits_equal(got, ref[name]), name
    grads, _ = fused_backward(g, x, y1, y2, y3, stats, weights, norms, True)
    for name in ("gW_conv", "gW_up"):
        got = grads[GRAD_KEYS.index(name)]
        assert _bits_equal(got, ref[name].view(got.shape)), name


def test_gradient_subsets_launch_only_what_is_asked():
    shape = (2, 35, 7, 12)
    x, weights, norms = operands(*shape, seed=5)
    g = torch.randn(x.shape).cuda()
    ref = unfused(x, weights, norms, True, g)
    (out, y1, y2, y3, stats), _ = fused_forward(x, weights, norms, True)
    for k in range(10):
        need = [j == k for j in range(10)]
        grads, bufs = fused_backward(g, x, y1, y2, y3, stats, weights, norms, True, need)
        got = grads[k]
        assert _bits_equal(got, ref[GRAD_KEYS[k]].view(got.shape)), GRAD_KEYS[k]
        assert all(gi is None for j, gi in enumerate(grads) if j != k)
        assert all(margins_intact(b) for b in bufs)


# ------------------------------------------------------------------------------------------------------------------------------
# the module
# ------------------------------------------------------------------------------------------------------------------------------
def _block(c, seed=0, momentum=0.1):
    torch.manual_seed(seed)
    b = Bottleneck(c)
    for m in b.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.momentum = momentum
            with torch.no_grad():
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.5, 1.5)
    return b


def _rel(a, b):
    return float((a.detach().double() - b.detach().double()).norm() / b.detach().double().norm().clamp_min(1e-30))


def _step(module, x, g, amp=False):
    for p in module.parameters():
        p.grad = None
    x = x.detach().clone().requires_grad_(True)
    with torch.autocast("cuda", enabled=amp):
        out = module(x)
    out.float().backward(g)
    grads = [x.grad] + [p.grad for p in module.parameters()]
    return out.float(), grads


@pytest.mark.parametrize("case", ["train", "eval", "train-amp", "train-momentum-none"])
def test_module_against_fp64(case):
    from fiery_b200.bottleneck import TensorCoreBottleneck
    training, amp = not case.startswith("eval"), case.endswith("amp")
    ref = _block(64, momentum=None if "none" in case else 0.1).cuda()
    ref.train(training)
    ours = TensorCoreBottleneck.from_module(copy.deepcopy(ref))
    f64 = copy.deepcopy(ref).double()
    x = torch.randn(6, 64, 40, 48, device="cuda")
    g = torch.randn(6, 64, 40, 48, device="cuda")
    r32 = copy.deepcopy(ref)
    o64, g64 = _step(f64, x.double(), g.double())
    o32, g32 = _step(r32, x, g, amp)
    o, gs = _step(ours, x, g, amp)
    assert o.dtype == torch.float32
    for got, want, base in zip([o] + gs, [o64] + g64, [o32] + g32):
        assert _rel(got, want) <= max(3 * _rel(base, want), 1e-3)
    for (name, b64), (_, b32), (_, b) in zip(f64.named_buffers(), r32.named_buffers(), ours.named_buffers()):
        if "num_batches_tracked" in name:
            assert int(b) == int(b64) == int(b32)
        else:
            assert _rel(b, b64) <= max(3 * _rel(b32, b64), 1e-3), name


def test_swapped_future_prediction_against_fp64():
    from fiery_b200 import install

    class Model(nn.Module):
        pass
    torch.manual_seed(0)
    fp = FuturePrediction(64, 32).cuda()
    model = Model()
    model.future_prediction = copy.deepcopy(fp)
    install.use_tensor_core_future_prediction(model)
    install.use_tensor_core_bottlenecks(model)
    x = torch.randn(2, 4, 32, 40, 48, device="cuda")
    h = torch.randn(2, 64, 40, 48, device="cuda")
    g = torch.randn(2, 4, 64, 40, 48, device="cuda")

    def run(m, dt):
        xi = x.to(dt).requires_grad_(True)
        out = m(xi, h.to(dt))
        out.backward(g.to(dt))
        return [out, xi.grad] + [p.grad for p in m.parameters()]
    r64 = run(copy.deepcopy(fp).double(), torch.float64)
    r32 = run(copy.deepcopy(fp), torch.float32)
    ours = run(model.future_prediction, torch.float32)
    for got, want, base in zip(ours, r64, r32):
        assert _rel(got, want) <= max(3 * _rel(base, want), 1e-3)


def test_repeats_graph_replay_and_compile_are_bit_identical():
    from fiery_b200.bottleneck import TensorCoreBottleneck
    ours = TensorCoreBottleneck.from_module(_block(70)).cuda()
    x = torch.randn(3, 70, 24, 36, device="cuda")
    g = torch.randn_like(x)
    first = _step(ours, x, g)
    for _ in range(2):
        torch.cuda.empty_cache()
        junk = torch.full((1 << 22,), float("nan"), device="cuda")   # recycled memory holds NaN
        del junk
        again = _step(ours, x, g)
        assert all(_bits_equal(a, b) for a, b in zip([first[0]] + first[1], [again[0]] + again[1]))
    ours.eval()
    static_x = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        ours(static_x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.no_grad():
        static_out = ours(static_x)
    eager = ours(x).detach()
    graph.replay()
    assert _bits_equal(static_out, eager)
    compiled = torch.compile(ours, backend="aot_eager")
    with torch.no_grad():
        assert _bits_equal(compiled(x), eager)


def test_opcheck():
    x, weights, norms = operands(2, 35, 8, 12, seed=2)
    args = (x.requires_grad_(True), *[w.requires_grad_(True) for w in weights], *norms, True, 1e-5)
    torch.library.opcheck(torch.ops.fiery_b200.bottleneck.default, args,
                          test_utils=("test_schema", "test_faketensor", "test_aot_dispatch_dynamic"))


def test_dispatches_no_aten_map_op():
    from fiery_b200.bottleneck import TensorCoreBottleneck
    ours = TensorCoreBottleneck.from_module(_block(64)).cuda()
    x = torch.randn(4, 64, 32, 32, device="cuda", requires_grad=True)
    _step(ours, x, torch.randn_like(x))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        out = ours(x)
        out.backward(torch.randn_like(out))
    names = {e.name for e in prof.events()}
    banned = [n for n in names if any(k in n for k in ("convolution", "cudnn", "batch_norm", "threshold"))
              or n in ("aten::relu", "aten::relu_", "aten::add")]
    assert not banned, banned


def test_forward_keeps_only_the_pre_norm_maps():
    from fiery_b200.bottleneck import TensorCoreBottleneck
    ours = TensorCoreBottleneck.from_module(_block(64)).cuda()
    x = torch.randn(4, 64, 64, 64, device="cuda", requires_grad=True)
    ours(x).sum().backward()                    # packs the weights, warms the caching allocator
    torch.cuda.synchronize()
    # the bytes the tensors ask for: memory_allocated() counts whole cached blocks, and the caching allocator hands out a block up to
    # 1 MiB larger than asked for when one is free, which depends on what ran earlier in the process
    before = torch.cuda.memory_stats()["requested_bytes.all.current"]
    out = ours(x)
    torch.cuda.synchronize()
    held = torch.cuda.memory_stats()["requested_bytes.all.current"] - before
    n, c, h, w = x.shape
    expect = 4 * n * h * w * (c + c // 2 + c // 2 + c)          # out, y1, y2, y3
    assert expect <= held <= expect + 4 * 4096                 # plus the per-channel statistics, rounded up by the allocator
    del out


def test_fallbacks_warn_once_and_match_the_reference():
    from fiery_b200 import _lib
    from fiery_b200.bottleneck import TensorCoreBottleneck
    _lib._warned.clear()
    ref = _block(64).cuda()
    x = torch.randn(2, 64, 12, 10, device="cuda")            # W % 4 != 0
    ours = TensorCoreBottleneck.from_module(copy.deepcopy(ref))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        a, b = ours(x), ours(x)
    assert sum("W = 10" in str(m.message) for m in w) == 1
    assert torch.allclose(a, copy.deepcopy(ref)(x), atol=1e-5) and torch.allclose(b, a, atol=1e-5)
    changed = TensorCoreBottleneck.from_module(copy.deepcopy(ref))
    changed.layers.dropout = nn.Dropout2d(0.5).eval()
    x4 = torch.randn(2, 64, 12, 16, device="cuda")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        changed(x4)
    assert any("dropout" in str(m.message) for m in w)
    synced = nn.SyncBatchNorm.convert_sync_batchnorm(TensorCoreBottleneck.from_module(copy.deepcopy(ref)))
    synced.eval()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        got = synced(x4)
    assert any("SyncBatchNorm" in str(m.message) for m in w)
    r = copy.deepcopy(ref).eval()
    assert torch.allclose(got, r(x4), atol=1e-4)
