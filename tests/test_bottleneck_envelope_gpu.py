"""The Bottleneck's kernels (fiery_bottleneck_*, fiery_bottleneck_sync_*_stage) element by element across their accepted envelope:
every forward stage and every gradient against the fp64 restatement of tests/_bottleneck_cases.py fed the kernels' own stage inputs,
each element within its bound, on every shape of ENVELOPE; the exact regime bit for bit; the TF32 rounding modes the header promises,
on ties; NaN and infinities; hard statistics; every backward subset; simulated groups; the module's variants against the C ABI bit for
bit; one run whose maps span more than 2^31 bytes.  Every output the C ABI writes lies between sentinel margins that are checked
unchanged, and every workspace starts filled with 0xFF bytes."""
from __future__ import annotations

import copy
import itertools

import pytest
import torch
import torch.nn as nn

from fiery_b200 import bottleneck as bk
from oracle.future_oracle import Bottleneck
from tests import _bottleneck_cases as bc
from tests import _spatial_gru_cases as gc
from tests._batch_norm_cases import merge_ranks
from tests.test_sync_bottleneck_gpu import _counting, _lockstep

pytestmark = pytest.mark.gpu

EPS = 1e-5
MARGINS = {}                     # stage -> the largest err / bound seen, reported at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report_margins():
    yield
    if MARGINS:
        print("\nlargest err/bound per stage: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(MARGINS.items())))


def _note(ratios, prefix=""):
    for k, (r, _) in ratios.items():
        MARGINS[prefix + k] = max(MARGINS.get(prefix + k, 0.0), r)


def _assert_within(ratios, what):
    bad = {k: v for k, v in ratios.items() if not (v[1] and v[0] <= 1.0)}
    assert not bad, (what, bad)


def _ids(s):
    return "x".join(str(v) for v in s)


def _grad_out(x, seed=7):
    return torch.randn(x.shape, generator=torch.Generator().manual_seed(seed)).to(x.device)


def _run(x, weights, norms, training, eps=EPS, g=None, label=""):
    """one forward (and with g a backward) through the C ABI, every stage and gradient checked against the restatement; returns
    (forward outputs, gradients)"""
    (out, y1, y2, y3, stats), bufs = bc.fused_forward(x, weights, norms, training, eps)
    stages, fw = bc.stage_ratios(bc.as_run(out, y1, y2, y3, stats), x, weights, norms, training, eps)
    _note(stages, label)
    _assert_within(stages, "forward stages")
    assert all(bc.margins_intact(b) for b in bufs), "forward wrote outside its outputs"
    if g is None:
        return (out, y1, y2, y3, stats), None
    grads, gbufs = bc.fused_backward(g, x, y1, y2, y3, stats, weights, norms, training, eps=eps)
    gr = bc.grad_ratios(fw, grads, weights, norms, g, training, eps)
    _note(gr, label + "d_")
    assert set(gr) == {k for k, t in zip(bc.GRAD_KEYS, grads) if t is not None}
    _assert_within(gr, "gradients")
    assert all(bc.margins_intact(b) for b in gbufs), "backward wrote outside its outputs"
    return (out, y1, y2, y3, stats), grads


# 1: every stage and every gradient at every shape of the envelope
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("shape", bc.ENVELOPE, ids=_ids)
def test_stages_and_gradients(shape, training):
    x, weights, norms = bc.operands(*shape, seed=sum(shape))
    _run(x, weights, norms, training, g=_grad_out(x))


# 2: the exact regime
def _dyadic(shape, scale, gen):
    return torch.randint(-1, 2, shape, generator=gen).double() * scale


def test_exact_regime_is_bit_exact():
    # integers times powers of two, small enough that every TF32 operand is exact and every fp32 sum is exact (y1 within 16 grains of
    # 1/2, y2 within 1152 of 1/8, the gradients likewise), and eval norms with scale exactly 1 and shift exactly 0: any summation order
    # and any operand rounding give the fp64 values
    maps, c, h, w = 3, 16, 9, 20
    m = c // 2
    gen = torch.Generator().manual_seed(1)
    x = _dyadic((maps, c, h, w), 1.0, gen)
    weights = [_dyadic((m, c, 1, 1), 0.5, gen), _dyadic((m, m, 3, 3), 0.25, gen), _dyadic((c, m, 1, 1), 0.5, gen)]
    norms = []
    for k in (m, m, c):
        norms += [torch.ones(k, dtype=torch.float64), torch.zeros(k, dtype=torch.float64), torch.zeros(k, dtype=torch.float64),
                  torch.ones(k, dtype=torch.float64)]
    g = _dyadic((maps, c, h, w), 0.25, gen)
    fw = bc.forward(x, weights, norms, False, 0.0, rounding=False)
    want, _ = bc.adjoint(fw, weights, norms, g, False, 0.0)
    fr = bc.forward(x, weights, norms, False, 0.0, rounding=True)
    wr, _ = bc.adjoint(fr, weights, norms, g, False, 0.0)
    for k in ("y1", "y2", "y3", "out"):                           # every rounding a no-op: the regime is exact
        assert torch.equal(fw["value"][k], fr["value"][k]), k
    assert all(torch.equal(want[k], wr[k]) for k in bc.GRAD_KEYS)
    cu = lambda ts: [t.float().cuda() for t in ts]                 # noqa: E731
    xc, wc, nc, gcu = x.float().cuda(), cu(weights), cu(norms), g.float().cuda()
    (out, y1, y2, y3, stats), bufs = bc.fused_forward(xc, wc, nc, False, 0.0)
    for k, got in (("y1", y1), ("y2", y2), ("y3", y3), ("out", out)):
        assert torch.equal(got.double().cpu(), fw["value"][k]), k
    grads, gbufs = bc.fused_backward(gcu, xc, y1, y2, y3, stats, wc, nc, False, eps=0.0)
    for k, got in zip(bc.GRAD_KEYS, grads):
        assert torch.equal(got.double().cpu(), want[k].reshape(got.shape)), k
    assert all(bc.margins_intact(b) for b in bufs + gbufs)


# 3: the rounding modes on ties
T11 = 2.0 ** -11


def _probe(c=4, h=1, w=4):
    """zero weights, identity eval norms (weight 1, bias 0, running mean 0, var 1, eps 0) at C channels: (weights, norms)"""
    m = c // 2
    weights = [torch.zeros(m, c, 1, 1), torch.zeros(m, m, 3, 3), torch.zeros(c, m, 1, 1)]
    norms = []
    for k in (m, m, c):
        norms += [torch.ones(k), torch.zeros(k), torch.zeros(k), torch.ones(k)]
    return weights, norms


def _probe_run(x, weights, norms, g=None):
    cu = lambda ts: [t.cuda() for t in ts]                         # noqa: E731
    (out, y1, y2, y3, stats), _ = bc.fused_forward(x.cuda(), cu(weights), cu(norms), False, 0.0)
    grads = None
    if g is not None:
        grads, _ = bc.fused_backward(g.cuda(), x.cuda(), y1, y2, y3, stats, cu(weights), cu(norms), False, eps=0.0)
    torch.cuda.synchronize()
    return (out, y1, y2, y3), grads


def test_rounding_of_the_3x3_and_up_projection_operands():
    # y1 = 1 + 2^-11 (x = 1 and 2^-11 on two channels): the 3x3 reads it rounded to nearest, ties away (1 + 2^-10); y2 = 1 + 3 2^-11
    # (the 3x3's reads of 1 + 2^-11 and 2^-11), a TF32 tie between 1 + 2^-10 and 1 + 2^-9: the up projection reads it truncated
    weights, norms = _probe(c=4)
    x = torch.zeros(1, 4, 1, 4)
    x[:, 0], x[:, 1] = 1.0, T11
    weights[0][0, 0], weights[0][0, 1] = 1.0, 1.0                  # y1[0] = 1 + 2^-11
    weights[0][1, 1] = 1.0                                         # y1[1] = 2^-11
    weights[1][0, 0, 1, 1] = 1.0                                   # y2[0] = rna(y1[0])
    weights[1][1, 0, 1, 1], weights[1][1, 1, 1, 1] = 1.0, 1.0      # y2[1] = rna(1 + 2^-11) + 2^-11
    weights[2][0, 1] = 1.0                                         # y3[0] = the up projection's read of y2[1]
    (out, y1, y2, y3), _ = _probe_run(x, weights, norms)
    assert bool((y1[:, 0] == 1 + T11).all())
    assert bool((y2[:, 0] == 1 + 2 * T11).all()), "the 3x3's activations: to nearest, ties away (rne and rz give 1)"
    # y2[1] = (1 + 2^-10) + 2^-11: a tie of TF32 again, between 1 + 2^-10 and 1 + 2^-9
    assert bool((y2[:, 1] == 1 + 3 * T11).all())
    assert bool((y3[:, 0] == 1 + 2 * T11).all()), "the up projection's activations: truncated (rna gives 1 + 2^-9)"


@pytest.mark.parametrize("sign", [1.0, -1.0], ids=["pos", "neg"])
def test_rounding_of_the_weight_gradient_operands(sign):
    # one pixel's output gradient: dy3 = g; da2 = W_up^T dy3 = s (1 + 2^-11) from g = s and s 2^-11 on two channels; dy2 = da2 (eval,
    # the masks open); the 3x3 weight gradient reads dy2 truncated: s 1 (away from zero gives s (1 + 2^-10), toward +inf gives 1 or
    # -(1 + 2^-10)).  The up projection's weight gradient reads dy3 = s (1 + 2^-11) on a third channel truncated as well.
    weights, norms = _probe(c=6)
    x = torch.zeros(1, 6, 1, 4)
    x[:, 0] = 1.0
    weights[0][:, 0] = 1.0                                         # y1 = 1 on the three mid channels
    weights[1][0, 0, 1, 1] = weights[1][1, 1, 1, 1] = 1.0          # y2[0] = y2[1] = 1
    weights[2][0, 0], weights[2][1, 0] = 1.0, 1.0                  # y3[0] = y3[1] = a2[0]: da2[0] = dy3[0] + dy3[1]
    weights[2][2, 1] = 1.0                                         # y3[2] = a2[1]
    g = torch.zeros(1, 6, 1, 4)
    g[0, 0, 0, 1], g[0, 1, 0, 1] = sign, sign * T11
    g[0, 2, 0, 2] = sign * (1 + T11)
    _, grads = _probe_run(x, weights, norms, g)
    gwc, gwu = grads[bc.GRAD_KEYS.index("gW_conv")].cpu(), grads[bc.GRAD_KEYS.index("gW_up")].cpu()
    assert float(gwc[0, 0, 1, 1]) == sign * 1.0, "the 3x3 weight gradient's output gradient: truncated"
    assert float(gwu[2, 1, 0, 0]) == sign * 1.0, "the up projection's weight gradient's output gradient: truncated"


# 4: non-finite values
@pytest.mark.parametrize("training", [False, True], ids=["eval", "train"])
@pytest.mark.parametrize("value", ["nan", "inf", "-inf", "nan_norm_weight"])
def test_non_finite_values(value, training):
    # every output and gradient non-finite exactly where the fp64 restatement is, the finite elements within their bounds: in eval a
    # non-finite x pixel reaches y1 there, y2 and y3 over its 3x3 neighbourhood (the prologue passes a NaN); in training it poisons
    # every statistic it reaches
    shape = (2, 24, 9, 20)
    x, weights, norms = bc.operands(*shape, seed=9)
    if value == "nan_norm_weight":
        norms[0][3] = float("nan")
    else:
        x[1, 5, 4, 7] = float(value)
    (out, y1, y2, y3, stats), _ = _run(x, weights, norms, training, g=_grad_out(x), label="nonfinite_")
    m = shape[1] // 2
    if value == "nan_norm_weight":
        assert not bool(torch.isnan(stats[:2 * m]).any())           # bn1's statistics are y1's
        if not training:
            bad = torch.isnan(y2).any(3).any(2).any(0)
            assert bool(bad.all())                                   # the NaN channel of a1 reaches every y2 channel
    elif value == "nan" and not training:
        assert bool(torch.isnan(y2[1, :, 3:6, 6:9]).all()) and int(torch.isnan(y2).sum()) == 9 * m
    elif value == "nan":
        assert bool(torch.isnan(stats).all())


# 5: hard statistics
@pytest.mark.parametrize("case", ["offset", "constant_channel", "eps0"])
def test_hard_statistics(case):
    shape = (3, 32, 17, 20)
    x, weights, norms = bc.operands(*shape, seed=11)
    weights = list(weights)
    eps = EPS
    if case == "offset":                                           # y1's mean >> its std
        x = x + 1e3
        weights[0] = weights[0].abs()
    elif case == "constant_channel":                               # y1[0] constant: var 0, scale weight / sqrt(eps)
        x[:, 0] = 0.75
        weights[0][0] = 0
        weights[0][0, 0] = 1.0
    else:
        eps = 0.0
    (_, _, _, _, stats), _ = _run(x, weights, norms, True, eps, g=_grad_out(x), label="hard_")
    if case == "constant_channel":
        assert float(stats[16]) == 0.0 and float(stats[0]) == 0.75


# 6: every backward subset
@pytest.mark.parametrize("shape", [(2, 35, 7, 12), (2, 70, 8, 16)], ids=["nchk1", "nchk2"])
def test_every_backward_subset_matches_the_full_call(shape):
    x, weights, norms = bc.operands(*shape, seed=13)
    g = _grad_out(x)
    (out, y1, y2, y3, stats), _ = bc.fused_forward(x, weights, norms, True)
    full, _ = bc.fused_backward(g, x, y1, y2, y3, stats, weights, norms, True)
    for need in itertools.product([False, True], repeat=10):
        grads, bufs = bc.fused_backward(g, x, y1, y2, y3, stats, weights, norms, True, need=need)
        for k, (nd, got, want) in enumerate(zip(need, grads, full)):
            assert (got is None) == (not nd)
            if nd:
                assert torch.equal(got, want), (need, bc.GRAD_KEYS[k])
        assert all(bc.margins_intact(b) for b in bufs), need


@pytest.mark.parametrize("world", [1, 3])
def test_every_backward_subset_gathers_as_sync_stages_says(world):
    shape = (4, 35, 7, 12)
    x, weights, norms = bc.operands(*shape, seed=14)
    params = [norms[i] for i in (0, 1, 4, 5, 8, 9)]
    g = _grad_out(x)
    sizes = [4] if world == 1 else [1, 0, 3]
    shards, gouts = torch.split(x, sizes), torch.split(g, sizes)
    fw = _lockstep([bk.sync_forward_stages(xr, *weights, params, EPS) for xr in shards])
    full = _lockstep([bk.sync_backward_stages(gr, xr, *f[1:5], *weights, params, EPS, [True] * 10)
                      for xr, gr, f in zip(shards, gouts, fw)])
    for need in itertools.product([False, True], repeat=10):
        calls = [[] for _ in shards]
        bw = _lockstep([_counting(bk.sync_backward_stages(gr, xr, *f[1:5], *weights, params, EPS, list(need)), cl)
                        for xr, gr, f, cl in zip(shards, gouts, fw, calls)])
        assert all(len(cl) == bk.sync_stages(need, params) for cl in calls), need
        for b, fb in zip(bw, full):
            for nd, got, want in zip(need, b, fb):
                assert (got is None) == (not nd) and (not nd or torch.equal(got, want)), need


# 7: simulated groups over the instantiation shapes of the envelope
GROUP_SHAPES = [s for s in bc.ENVELOPE if s[0] * s[2] * s[3] < 200_000 and s[0] < 300]


def _sizes(maps):
    return [0, 1] if maps == 1 else [1, 0, maps - 1]              # an empty rank and a one-map rank


@pytest.mark.parametrize("shape", GROUP_SHAPES, ids=_ids)
def test_simulated_groups(shape):
    maps, c, h, w = shape
    m = c // 2
    x, weights, norms = bc.operands(*shape, seed=sum(shape) + 1)
    params = [norms[i] for i in (0, 1, 4, 5, 8, 9)]
    g = _grad_out(x, seed=3)
    sizes = _sizes(maps)
    shards, gouts = torch.split(x, sizes), torch.split(g, sizes)
    fw = _lockstep([bk.sync_forward_stages(xr, *weights, params, EPS) for xr in shards])
    bw = _lockstep([bk.sync_backward_stages(gr, xr, *f[1:5], *weights, params, EPS, [True] * 10)
                    for xr, gr, f in zip(shards, gouts, fw)])
    for f in fw:                                                   # every rank the group's statistics and counts, bit for bit
        assert torch.equal(f[4], fw[0][4]) and torch.equal(f[5], torch.full((3,), float(maps * h * w), dtype=torch.float64,
                                                                             device=x.device))
    # the ranks together are the whole batch's computation with the group's statistics: each stage and gradient within the
    # restatement's bounds (the weight and norm gradients are the ranks' own sums, added up)
    cat = lambda k: torch.cat([f[k] for f in fw])                   # noqa: E731
    run = bc.as_run(cat(0), cat(1), cat(2), cat(3), fw[0][4])
    stages, rfw = bc.stage_ratios(run, x, weights, norms, True, EPS)
    _note(stages, "group_")
    _assert_within(stages, "forward stages")
    grads = [torch.cat([b[0] for b in bw])] + [sum(b[k] for b in bw) for k in range(1, 10)]
    gr = bc.grad_ratios(rfw, grads, weights, norms, g, True, EPS)
    _note(gr, "group_d_")
    _assert_within(gr, "gradients")
    # the merge restated: each rank's fp64 (n, mean, M2) of its y merged in rank order, within the statistics' bounds
    for i, (o, k) in enumerate(((0, m), (2 * m, m), (4 * m, c))):
        trip = []
        for f in fw:
            y = f[1 + i].double()
            n = y.shape[0] * h * w
            mean = y.mean((0, 2, 3)) if n else torch.zeros(k, dtype=torch.float64, device=x.device)
            m2 = ((y - mean.view(1, -1, 1, 1)) ** 2).sum((0, 2, 3)) if n else torch.zeros_like(mean)
            trip.append(torch.stack([torch.full_like(mean, float(n)), mean, m2], 1).cpu().numpy())
        nn_, mm, mm2 = merge_ranks(trip, contracted=True)
        for got, want, bound in ((fw[0][4][o:o + k], mm, rfw["bound"][f"mean{i + 1}"]),
                                 (fw[0][4][o + k:o + 2 * k], mm2 / nn_, rfw["bound"][f"var{i + 1}"])):
            r, same = gc.excess(got.cpu(), torch.from_numpy(want), bound.cpu())
            assert same and r <= 1.0, (i, r)


# 8: module variants against the C ABI called with the arguments each implies
def _block(c, seed=0, affine=True, track=True, momentum=0.1, eps=1e-5):
    torch.manual_seed(seed)
    b = Bottleneck(c)
    for name in ("abn_down_project", "abn", "abn_up_project"):
        seq = getattr(b.layers, name)
        k = seq[0].num_features
        seq[0] = nn.BatchNorm2d(k, eps=eps, momentum=momentum, affine=affine, track_running_stats=track)
        with torch.no_grad():
            if affine:
                seq[0].weight.uniform_(0.5, 1.5)
                seq[0].bias.uniform_(-0.3, 0.3)
            if track:
                seq[0].running_mean.uniform_(-0.2, 0.2)
                seq[0].running_var.uniform_(0.5, 1.5)
    return b.cuda()


def _abi_args(block):
    """(weights, the 12 norm parameters, batch statistics, eps) the module passes for this block"""
    layers = block.layers
    bns = [layers.abn_down_project[0], layers.abn[0], layers.abn_up_project[0]]
    batch = bns[0].training or bns[0].running_mean is None
    norms = []
    for bn in bns:
        norms += [bn.weight, bn.bias, None if batch else bn.running_mean, None if batch else bn.running_var]
    weights = [layers.conv_down_project.weight, layers.conv.weight, layers.conv_up_project.weight]
    return [t.detach().clone() for t in weights], [t.detach().clone() if t is not None else None for t in norms], batch, bns[0].eps


def _bn_update(rm, rv, mean, var, n, momentum, tracked):
    f = 1.0 / tracked if momentum is None else momentum
    return rm * (1 - f) + mean * f, rv * (1 - f) + var * (n / (n - 1)) * f


VARIANTS = ["c2", "c17", "c35", "c70", "c128", "affine_false", "untracked_train", "untracked_eval", "momentum_none", "eps0",
            "eps1e-3", "channels_last", "misaligned", "fp16_autocast"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_module_variants_match_the_c_abi(variant):
    c = int(variant[1:]) if variant[0] == "c" and variant[1:].isdigit() else 34
    ref = _block(c, affine=variant != "affine_false", track=not variant.startswith("untracked"),
                 momentum=None if variant == "momentum_none" else 0.1,
                 eps={"eps0": 0.0, "eps1e-3": 1e-3}.get(variant, 1e-5))
    if variant == "untracked_eval":
        ref.eval()
    ours = bk.TensorCoreBottleneck.from_module(copy.deepcopy(ref))
    weights, norms, batch, eps = _abi_args(ours)
    before = [b.clone() for b in ours.buffers()]
    x = torch.randn(3, c, 9, 20, device="cuda")
    g = torch.randn(3, c, 9, 20, device="cuda")
    xin = x
    if variant == "channels_last":
        xin = x.contiguous(memory_format=torch.channels_last)
    elif variant == "misaligned":
        buf = torch.empty(x.numel() + 1, device="cuda")
        xin = buf[1:].view(x.shape)
        xin.copy_(x)
        assert xin.data_ptr() % 16
    elif variant == "fp16_autocast":
        xin = x.half()
    xr = xin.requires_grad_(True) if variant == "misaligned" else xin.detach().clone().requires_grad_(True)
    with torch.autocast("cuda", enabled=variant == "fp16_autocast"):
        out = ours(xr)
    out.backward(g)
    xf = x if variant == "misaligned" else xin.detach().float().contiguous()
    (o, y1, y2, y3, stats), _ = bc.fused_forward(xf, weights, norms, batch, eps)
    grads, _ = bc.fused_backward(g, xf, y1, y2, y3, stats, weights, norms, batch, eps=eps)
    assert out.dtype == torch.float32 and torch.equal(out, o)
    assert xr.grad.dtype == xin.dtype and torch.equal(xr.grad, grads[0].to(xin.dtype))
    layers = ours.layers
    for conv, gw in zip((layers.conv_down_project, layers.conv, layers.conv_up_project), grads[1:4]):
        assert torch.equal(conv.weight.grad, gw.view(conv.weight.shape))
    bns = [layers.abn_down_project[0], layers.abn[0], layers.abn_up_project[0]]
    for i, bn in enumerate(bns):
        if bn.affine:
            assert torch.equal(bn.weight.grad, grads[4 + 2 * i]) and torch.equal(bn.bias.grad, grads[5 + 2 * i])
        else:
            assert grads[4 + 2 * i] is None or bn.weight is None
    m = c // 2
    for i, (bn, (o_, k)) in enumerate(zip(bns, bk._stats_slices(m, c))):
        if not bn.track_running_stats:
            assert bn.running_mean is None
            continue
        rm0, rv0, nbt0 = before[3 * i], before[3 * i + 1], before[3 * i + 2]
        if bn.training:
            assert int(bn.num_batches_tracked) == int(nbt0) + 1
            want_m, want_v = _bn_update(rm0, rv0, stats[o_:o_ + k], stats[o_ + k:o_ + 2 * k], 3 * 9 * 20, bn.momentum,
                                        int(bn.num_batches_tracked))
            torch.testing.assert_close(bn.running_mean, want_m, rtol=1e-6, atol=1e-7)
            torch.testing.assert_close(bn.running_var, want_v, rtol=1e-6, atol=1e-7)


def test_sgd_steps_and_load_state_dict():
    # three SGD steps; after each in-place step and after load_state_dict the swapped module computes what a fresh swap of the same
    # weights (a new pack) computes, bit for bit, so the pack cache follows the updates; the running statistics count every step
    ref = _block(34, seed=2)
    ours = bk.TensorCoreBottleneck.from_module(ref)
    opt = torch.optim.SGD(ours.parameters(), lr=0.05)
    x = torch.randn(3, 34, 9, 20, device="cuda")

    def fresh_eval():
        f = bk.TensorCoreBottleneck.from_module(copy.deepcopy(ref)).eval()
        ours.eval()
        want, got = f(x), ours(x)
        ours.train()
        return torch.equal(got, want)

    for step in range(3):
        opt.zero_grad()
        (ours(x) * x.cos()).sum().backward()
        opt.step()
        assert fresh_eval(), step
    assert int(ours.layers.abn[0].num_batches_tracked) == 3
    ours.load_state_dict(_block(34, seed=5).state_dict())
    assert fresh_eval()


# 9: one run past 2^31 bytes
def test_maps_past_two_gigabytes():
    maps, c, h, w = 105, 128, 200, 200
    m = c // 2
    big, small = maps * c * h * w * 4, maps * m * h * w * 4
    assert big > 2 ** 31
    # x, out, y3, grad_out, grad_x (C channels), y1, y2 (M), the backward workspace (dy3 and two M-channel buffers), slack for the
    # per-map restatement
    need = 5 * big + 2 * small + (big + 2 * small) + (2 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    _, weights, norms = bc.operands(1, c, 4, 4, seed=17)
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(maps, c, h, w, device="cuda", generator=gen)
    # training forward: the statistics over the whole batch in fp64 on the device, the per-map stages with them on the first and
    # last map
    (out, y1, y2, y3, stats), bufs = bc.fused_forward(x, weights, norms, True)
    run_stats = stats.clone()
    for i, (o, k, y) in enumerate(((0, m, y1), (2 * m, m, y2), (4 * m, c, y3))):
        s1 = sum(y[j:j + 8].double().sum((0, 2, 3)) for j in range(0, maps, 8))
        mean = s1 / (maps * h * w)
        s2 = sum(((y[j:j + 8].double() - mean.view(1, -1, 1, 1)) ** 2).sum((0, 2, 3)) for j in range(0, maps, 8))
        sa = sum(y[j:j + 8].double().abs().sum((0, 2, 3)) for j in range(0, maps, 8)) / (maps * h * w)
        sd = sum((y[j:j + 8].double() - mean.view(1, -1, 1, 1)).abs().sum((0, 2, 3)) for j in range(0, maps, 8)) / (maps * h * w)
        var = s2 / (maps * h * w)
        em = bc.BN_SUM * bc.SUM * sa
        for got, want, bound in ((stats[o:o + k], mean, em), (stats[o + k:o + 2 * k], var, 2 * bc.BN_SUM * bc.SUM * var + 4 * em * sd + em ** 2)):
            r, same = gc.excess(got, want, bound)
            MARGINS["large_stats"] = max(MARGINS.get("large_stats", 0.0), r)
            assert same and r <= 1.0, (i, r)
    for j in (0, maps - 1):
        sl = slice(j, j + 1)
        stages, _ = bc.stage_ratios(bc.as_run(out[sl], y1[sl], y2[sl], y3[sl], run_stats), x[sl], weights, norms, True, EPS)
        stages = {k: v for k, v in stages.items() if k in ("y1", "y2", "y3", "out")}
        _note(stages, "large_")
        _assert_within(stages, ("map", j))
    assert all(bc.margins_intact(b) for b in bufs)
    del out, y1, y2, y3, bufs
    # eval forward and backward: per-map stages and dx on the first and last map, each weight gradient against the sum of the per-map
    # adjoints (an eval norm's backward is per element)
    g = torch.randn(maps, c, h, w, device="cuda", generator=gen)
    (out, y1, y2, y3, stats), _ = bc.fused_forward(x, weights, norms, False)
    grads, gbufs = bc.fused_backward(g, x, y1, y2, y3, stats, weights, norms, False, need=(True, True, True, True) + (False,) * 6)
    want = {k: 0 for k in ("gW_down", "gW_conv", "gW_up")}
    bound = dict(want)
    for j in range(maps):
        sl = slice(j, j + 1)
        stages, fw = bc.stage_ratios(bc.as_run(out[sl], y1[sl], y2[sl], y3[sl], stats), x[sl], weights, norms, False, EPS)
        if j in (0, maps - 1):
            _note(stages, "large_")
            _assert_within(stages, ("map", j))
        wj, bj = bc.adjoint(fw, weights, [t.double() for t in norms], g[sl].double(), False, EPS, maps_total=maps)
        if j in (0, maps - 1):
            r = {"dx": gc.excess(grads[0][sl], wj["dx"], bj["dx"])}
            _note(r, "large_d_")
            _assert_within(r, ("dx", j))
        for k in want:
            want[k] = want[k] + wj[k]
            bound[k] = bound[k] + bj[k]
    r = {k: gc.excess(grads[bc.GRAD_KEYS.index(k)], want[k].reshape(grads[bc.GRAD_KEYS.index(k)].shape),
                      bound[k].reshape(grads[bc.GRAD_KEYS.index(k)].shape)) for k in want}
    _note(r, "large_d_")
    _assert_within(r, "weight gradients")
    assert all(bc.margins_intact(b) for b in gbufs)
