"""The output head through the C ABI across its accepted shapes and values, as tests/test_bottleneck_envelope_gpu.py does for the
Bottleneck: every output and gradient element by element against the fp64 restatement of tests/_output_head_cases.py fed the run's
statistics, each within its bound, on every case of its ENVELOPE table, the ring-wrapping cases of the device's SM count and the shipped
shapes; the TF32 rounding contract bit for bit on ties; NaN and infinities; hard statistics; FusedOutputHead's variants against the C
ABI bit for bit; and y past 2^31 bytes in eval and in training.  Every output the C ABI writes lies between sentinel margins that are
checked unchanged, and every workspace starts filled with 0xFF bytes.  H100 only."""
from __future__ import annotations

import copy
import warnings

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from fiery_b200 import _lib
from fiery_b200 import decoder as dec
from oracle import decoder_oracle as DO
from tests import _output_head_cases as oc
from tests import _spatial_gru_cases as gc

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


def _grad_out(maps, n, h, w, seed=7):
    return torch.randn((maps, n, h, w), generator=torch.Generator().manual_seed(seed)).cuda()


def _run(y, w1, b1, norm, training, eps=EPS, g=None, label="", keys=None):
    """one forward (and with g a backward) through the C ABI, the outputs and gradients (those in ``keys``, default all) checked against
    the restatement; returns ((out, mean, var), gradients)"""
    (out, mean, var), bufs = oc.fused_forward(y, w1, b1, norm, training, eps)
    stages, fw = oc.stage_ratios((out, mean, var), y, w1, b1, norm, training, eps)
    stages = {k: v for k, v in stages.items() if keys is None or k in keys}
    _note(stages, label)
    _assert_within(stages, "forward")
    assert all(oc.margins_intact(b) for b in bufs), "forward wrote outside its outputs"
    if g is None:
        return (out, mean, var), None
    grads, gbufs = oc.fused_backward(g, y, mean, var, w1, b1, norm, training, eps=eps)
    gr = oc.grad_ratios(fw, grads, w1, b1, norm, g, training, eps)
    assert set(gr) == {k for k, t in zip(oc.GRAD_KEYS, grads) if t is not None}
    gr = {k: v for k, v in gr.items() if keys is None or k in keys}
    _note(gr, label + "d_")
    _assert_within(gr, "gradients")
    assert all(oc.margins_intact(b) for b in gbufs), "backward wrote outside its outputs"
    return (out, mean, var), grads


def _case(case, seed=None):
    maps, c, n, h, w, training = case
    y, w1, b1, norm = oc.operands(maps, c, n, h, w, seed=sum(case) if seed is None else seed)
    _run(y, w1, b1, norm, training, g=_grad_out(maps, n, h, w, seed=c + n))


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# 1: the envelope table, the ring-wrapping cases and the shipped shapes
@pytest.mark.parametrize("case", oc.ENVELOPE, ids=lambda c: "x".join(str(v) for v in c[:5]) + ("_train" if c[5] else "_eval"))
def test_envelope_table(case):
    _case(case)


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("kp", oc.KPADS, ids=lambda k: f"kpad{k}")
def test_every_cta_wraps_its_ring(kp, training):
    # as many 100 x 130 maps as make every persistent CTA of this device use each ring stage twice, so every mbarrier phase flips and
    # every CTA rewrites its row table for a tile of another map
    sms = _sms()
    case = oc.wrap_case(kp, sms)[:5] + (training,)
    r = oc.reach(case, sms)
    assert r["ring_wrap"] and r["frame_change"], r
    _case(case)


@pytest.mark.parametrize("case", oc.SHIPPED, ids=lambda c: f"{c[0]}maps_n{c[2]}")
def test_shipped_shapes(case):
    assert oc.reach(case, _sms())["wg1_valid"] == 0
    _case(case)



CHANNELS = (1, 8, 63, 64, 65, 128)
# (X, Y): 4 pixels, one short of / at / one past a 128-pixel tile, at / past a 4096-pixel piece
GRIDS = ((1, 4), (4, 31), (4, 32), (4, 33), (64, 64), (41, 100))
CASES = [(c, n, GRIDS[(i + n) % len(GRIDS)], (i + n) % 2 == 0) for i, c in enumerate(CHANNELS) for n in range(1, 9)]


@pytest.mark.parametrize("c,n,grid,training", CASES, ids=lambda v: str(v))
def test_envelope(c, n, grid, training):
    h, w = grid
    maps = 3
    y, w1, b1, norm = oc.operands(maps, c, n, h, w, seed=c * 10 + n)
    (out, mean, var), bufs = oc.fused_forward(y, w1, b1, norm, training)
    assert all(oc.margins_intact(b) for b in bufs)
    ratios, fw = oc.stage_ratios((out, mean, var), y, w1, b1, norm, training, 1e-5)
    assert all(same and r <= 1.0 for r, same in ratios.values()), ratios
    g = torch.randn_like(out)
    grads, bufs = oc.fused_backward(g, y, mean, var, w1, b1, norm, training)
    assert all(oc.margins_intact(b) for b in bufs)
    r = oc.grad_ratios(fw, grads, w1, b1, norm, g, training, 1e-5)
    assert all(same and v <= 1.0 for v, same in r.values()), r


def test_y_past_2_31_bytes():
    """eval: every map is independent of the others, so the last map of a > 2 GiB y must come out bit for bit as on its own"""
    maps, c, n, h, w = 19, 128, 2, 480, 480                # 2.24e9 bytes
    torch.manual_seed(0)
    y = torch.randn(maps, c, h, w, device="cuda")
    _, w1, b1, norm = oc.operands(1, c, n, 4, 4)
    (out, mean, var), _ = oc.fused_forward(y, w1, b1, norm, False)
    g = torch.randn_like(out)
    grads, _ = oc.fused_backward(g, y, mean, var, w1, b1, norm, False, need=(True, False, False, False, False))
    gy = grads[0][-1:].clone()
    del grads
    last = y[-1:].clone()
    del y
    (out1, _, _), _ = oc.fused_forward(last, w1, b1, norm, False)
    assert torch.equal(out[-1:], out1)
    g1, _ = oc.fused_backward(g[-1:].contiguous(), last, mean, var, w1, b1, norm, False, need=(True, False, False, False, False))
    assert torch.equal(gy, g1[0])


# 2: the rounding contract, bit for bit on ties.  Eval with running mean 0, running var 1, weight 1, bias 0 and eps 0, so a = relu(y).
T11, T20 = 2.0 ** -11, 2.0 ** -20


def _probe_operands():
    """C = 2, n = 3, 1 x 8 pixels: y = 1 + 2^-11 on channel 0's pixels 0..3 and -1 on 4..7 (a = 0 there), channel 1 zero; W1 rows
    +-(1 + 2^-11) on channel 0 and a zero row; b1 = 2^-20, 2^-20, 1 + 2^-20"""
    y = torch.zeros(1, 2, 1, 8)
    y[0, 0, 0, :4], y[0, 0, 0, 4:] = 1 + T11, -1.0
    w1 = torch.zeros(3, 2, 1, 1)
    w1[0, 0], w1[1, 0] = 1 + T11, -(1 + T11)
    b1 = torch.tensor([T20, T20, 1 + T20])
    norm = [torch.ones(2), torch.zeros(2), torch.zeros(2), torch.ones(2)]
    return y.cuda(), w1.cuda(), b1.cuda(), [t.cuda() for t in norm]


def test_rounding_contract_bit_exact():
    y, w1, b1, norm = _probe_operands()
    (out, mean, var), _ = oc.fused_forward(y, w1, b1, norm, False, 0.0)
    out = out.cpu()
    # W1 rounded to nearest with ties away: 1 + 2^-11 is the tie between 1 and 1 + 2^-10 (to nearest even and toward zero give 1);
    # a = 1 + 2^-11 truncated to 1 (to nearest gives 1 + 2^-10 and a product of 1 + 2^-9 + 2^-20); b1 added in fp32
    assert bool((out[0, 0, 0, :4] == 1 + 2 * T11 + T20).all()), out[0, 0]
    assert bool((out[0, 1, 0, :4] == -(1 + 2 * T11) + T20).all()), out[0, 1]
    assert bool((out[0, :2, 0, 4:] == T20).all())
    assert bool((out[0, 2] == 1 + T20).all()), "b1 is not rounded to TF32 (it would give 1)"
    # one output gradient per pixel: g[0] = 1 at pixel 1, g[1] = 1 at pixel 2, g[2] = 1 at pixel 5 (masked)
    g = torch.zeros(1, 3, 1, 8)
    g[0, 0, 0, 1], g[0, 1, 0, 2], g[0, 2, 0, 5] = 1.0, 1.0, 1.0
    grads, _ = oc.fused_backward(g.cuda(), y, mean, var, w1, b1, norm, False, eps=0.0)
    gy, gbw, gbb, gw, gb = (t.cpu() for t in grads)
    assert float(gy[0, 0, 0, 1]) == 1 + T11 and float(gy[0, 0, 0, 2]) == -(1 + T11), "da uses the fp32 W1 (the packed one is 1 + 2^-10)"
    assert float(gy[0, 0, 0, 5]) == 0.0 and bool((gy[0, 1] == 0).all())
    assert float(gw[0, 0]) == 1 + T11 and float(gw[1, 0]) == 1 + T11, "dW1 uses the unrounded a (truncated it is 1)"
    assert bool((gw[:, 1] == 0).all()) and float(gw[2, 0]) == 0.0
    assert gb.tolist() == [1.0, 1.0, 1.0]
    # and every output and gradient is the restatement's exactly: each is one product or a sum of exact terms
    fw = oc.forward(y.double(), w1, b1, [t.double() for t in norm], False, 0.0)
    assert torch.equal(out.double(), fw["value"]["out"].cpu())
    want, _ = oc.adjoint(fw, w1, b1, [t.double() for t in norm], g.cuda().double(), False, 0.0)
    for k, got in zip(oc.GRAD_KEYS, (gy, gbw, gbb, gw, gb)):
        assert torch.equal(got.double(), want[k].cpu().reshape(got.shape)), k


# 3: non-finite values
NONFINITE = ["y_nan", "y_inf", "y_neg_inf", "bn_weight_nan", "w1_inf", "b1_nan", "grad_out_nan"]


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("value", NONFINITE)
def test_non_finite_values(value, training):
    # every output and gradient non-finite exactly where the restatement's is, the finite elements within their bounds.  In eval a
    # non-finite y pixel reaches that pixel's outputs; in training it poisons its channel's statistics and so every output.  A NaN norm
    # weight makes its channel's a NaN everywhere; an infinite W1 entry its output row and its channel's da; a NaN b1 its output row; a
    # NaN grad_out its pixel's da in every channel (in training every unmasked channel's dy) and its row of dW1 and db1.
    maps, c, n, h, w = 2, 24, 3, 9, 20
    y, w1, b1, norm = oc.operands(maps, c, n, h, w, seed=9)
    g = _grad_out(maps, n, h, w, seed=10)
    if value.startswith("y_"):
        y[1, 5, 4, 7] = {"y_nan": float("nan"), "y_inf": float("inf"), "y_neg_inf": float("-inf")}[value]
    elif value == "bn_weight_nan":
        norm[0][3] = float("nan")
    elif value == "w1_inf":
        w1[1, 6] = float("inf")
    elif value == "b1_nan":
        b1[2] = float("nan")
    else:
        g[1, 0, 4, 7] = float("nan")
    (out, mean, var), grads = _run(y, w1, b1, norm, training, g=g, label="nonfinite_")
    assert not all(bool(torch.isfinite(t).all()) for t in [out, mean, var] + [t for t in grads if t is not None])
    if value == "grad_out_nan":
        assert bool(torch.isnan(grads[3][0]).all()) and bool(torch.isnan(grads[4][0])) and bool(torch.isfinite(grads[4][1:]).all())


def test_zero_running_variance_in_eval():
    # running_var + eps = 0 on one channel: scale = weight / 0 = inf and shift = bias - mean * inf, so the kernels' fmaf(scale, y, shift)
    # is NaN where y > 0 (inf - inf) and -inf where y < 0 (a = 0), while torch's (y - mean) * invstd is +-inf with a NaN only at y == mean.
    # This is the one place the kernels and torch's batch norm disagree; the restatement follows the kernels' formula.  The norm
    # gradients are left out: the kernels form them as S2 / sqrt(var + eps), the restatement term by term, and with an infinite
    # invstd the two differ in which non-finite value they give.
    maps, c, n, h, w = 2, 8, 2, 4, 8
    y, w1, b1, norm = oc.operands(maps, c, n, h, w, seed=12)
    norm[2][1], norm[3][1], norm[0][1] = 0.3, 0.0, 1.0
    g = _grad_out(maps, n, h, w, seed=13)
    (out, _, _), grads = _run(y, w1, b1, norm, False, eps=0.0, g=g, label="zero_var_",
                             keys=("out", "mean", "var", "gy", "gW", "gb"))
    assert bool(torch.isnan(out).any())


# 4: hard statistics
@pytest.mark.parametrize("case", ["offset", "constant_channel", "eps0"])
def test_hard_statistics(case):
    maps, c, n, h, w = 3, 32, 2, 17, 20
    y, w1, b1, norm = oc.operands(maps, c, n, h, w, seed=11)
    eps = EPS
    if case == "offset":                                           # mean 1e3 over a std of 0.5
        y = y + 1e3
    elif case == "constant_channel":                               # var 0: scale weight / sqrt(eps)
        y[:, 0] = 0.75
    else:
        eps = 0.0
    (_, mean, var), _ = _run(y, w1, b1, norm, True, eps, g=_grad_out(maps, n, h, w), label="hard_")
    if case == "constant_channel":
        assert float(mean[0]) == 0.75 and float(var[0]) == 0.0


# 5: FusedOutputHead's variants against the C ABI, bit for bit
def _head(c, n, sigmoid=False, seed=0, affine=True, track=True, momentum=0.1, eps=1e-5):
    torch.manual_seed(seed)
    head = DO.output_head(c, n, sigmoid)
    head[1] = nn.BatchNorm2d(c, eps=eps, momentum=momentum, affine=affine, track_running_stats=track)
    with torch.no_grad():
        if affine:
            head[1].weight.uniform_(0.5, 1.5), head[1].bias.uniform_(-0.3, 0.3)
        if track:
            head[1].running_mean.uniform_(-0.2, 0.2), head[1].running_var.uniform_(0.5, 1.5)
    return head.cuda()


def _deterministic():
    return torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True, allow_tf32=torch.backends.cudnn.allow_tf32)


VARIANTS = ([f"c{c}_n{n}" for c in (2, 17, 64, 128) for n in ("1s", "2", "8")] +
            ["affine_false", "untracked_train", "untracked_eval", "momentum_none", "eps0", "eps1e-3", "channels_last", "fp16_autocast",
             "bf16_autocast"])


@pytest.mark.parametrize("variant", VARIANTS)
def test_module_variants_match_the_c_abi(variant):
    c, n, sigmoid = 24, 2, False
    if variant.startswith("c") and "_n" in variant:
        c, n, sigmoid = int(variant[1:variant.index("_")]), int(variant[variant.index("_n") + 2]), variant.endswith("s")
    ref = _head(c, n, sigmoid, affine=variant != "affine_false", track=not variant.startswith("untracked"),
                momentum=None if variant == "momentum_none" else 0.1, eps={"eps0": 0.0, "eps1e-3": 1e-3}.get(variant, 1e-5))
    if variant == "untracked_eval":
        ref.eval()
    ours = dec.FusedOutputHead.from_module(copy.deepcopy(ref))
    conv, bn, conv1 = ours[0], ours[1], ours[3]
    batch = bn.training or bn.running_mean is None
    norm = [t.detach().clone() if t is not None else None for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var)]
    nbt0 = int(bn.num_batches_tracked) if bn.track_running_stats else None
    dt16 = {"fp16_autocast": torch.float16, "bf16_autocast": torch.bfloat16}.get(variant)
    x = torch.randn(3, c, 9, 20, device="cuda")
    g = torch.randn(3, n, 9, 20, device="cuda")
    if variant == "channels_last":
        x = x.contiguous(memory_format=torch.channels_last)
    xr = x.clone().requires_grad_(True)
    with _deterministic(), torch.autocast("cuda", dtype=dt16 or torch.float16, enabled=dt16 is not None):
        out = ours(xr)
    with _deterministic():
        out.backward(g)
    # the same 3x3 on the same input, the C ABI on its output, the sigmoid and the 3x3's backward as autograd runs them
    xc, wc = x.clone().requires_grad_(True), conv.weight.detach().clone().requires_grad_(True)
    with _deterministic(), torch.autocast("cuda", dtype=dt16 or torch.float16, enabled=dt16 is not None):
        y = F.conv2d(xc, wc, None, conv.stride, conv.padding, conv.dilation, conv.groups)
    yf = y.detach().float().contiguous()
    (o, mean, var), _ = oc.fused_forward(yf, conv1.weight.detach(), conv1.bias.detach(), norm, batch, bn.eps)
    go = g
    if sigmoid:
        oc_ = o.clone().requires_grad_(True)
        s = torch.sigmoid(oc_)
        s.backward(g)
        o, go = s.detach(), oc_.grad
    grads, _ = oc.fused_backward(go, yf, mean, var, conv1.weight.detach(), conv1.bias.detach(), norm, batch, eps=bn.eps)
    with _deterministic():
        y.backward(grads[0].to(y.dtype))
    assert out.dtype == torch.float32 and torch.equal(out, o)
    assert torch.equal(xr.grad, xc.grad) and torch.equal(conv.weight.grad, wc.grad)
    assert torch.equal(conv1.weight.grad, grads[3].view(conv1.weight.shape)) and torch.equal(conv1.bias.grad, grads[4])
    if bn.affine:
        assert torch.equal(bn.weight.grad, grads[1]) and torch.equal(bn.bias.grad, grads[2])
    if not bn.track_running_stats:
        assert bn.running_mean is None and bn.running_var is None
    elif bn.training:
        assert int(bn.num_batches_tracked) == nbt0 + 1
        (wm, bm), (wv, bv) = oc.running_update(norm[2], norm[3], mean, var, 3 * 9 * 20, bn.momentum, nbt0 + 1)
        for got, want, bound in ((bn.running_mean, wm, bm), (bn.running_var, wv, bv)):
            r, same = gc.excess(got, want, bound)
            assert same and r <= 1.0, r


def test_misaligned_y_through_the_operator():
    # a y whose address is 4 bytes past a 16-byte boundary is copied once to an aligned tensor: the same results as the aligned y
    c, n = 24, 2
    y, w1, b1, norm = oc.operands(3, c, n, 9, 20, seed=21)
    buf = torch.empty(y.numel() + 1, device="cuda")
    ym = buf[1:].view(y.shape)
    ym.copy_(y)
    assert ym.data_ptr() % 16
    leaves = [t.clone().requires_grad_(True) for t in (w1, b1, norm[0], norm[1])]
    ym.requires_grad_(True)
    out, mean, var = torch.ops.fiery_b200.output_head(ym, leaves[0], leaves[1], leaves[2], leaves[3], None, None, True, EPS)
    g = _grad_out(3, n, 9, 20)
    out.backward(g)
    (o, m, v), _ = oc.fused_forward(y, w1, b1, norm, True)
    assert torch.equal(out, o) and torch.equal(mean, m) and torch.equal(var, v)
    grads, _ = oc.fused_backward(g, y, m, v, w1, b1, norm, True)
    assert torch.equal(ym.grad, grads[0]) and torch.equal(leaves[2].grad, grads[1]) and torch.equal(leaves[3].grad, grads[2])
    assert torch.equal(leaves[0].grad, grads[3].view(w1.shape)) and torch.equal(leaves[1].grad, grads[4])


def test_pixels_not_a_multiple_of_4_run_the_reference_with_one_warning():
    ref = _head(16, 2, seed=3)
    ours = dec.FusedOutputHead.from_module(copy.deepcopy(ref))
    for key in [k for k in _lib._warned if k[0] == "output_head"]:
        _lib._warned.discard(key)
    x = torch.randn(2, 16, 7, 9, device="cuda")
    with warnings.catch_warnings(record=True) as caught, _deterministic():
        warnings.simplefilter("always")
        for _ in range(2):
            xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
            oa, ob = ours(xa), ref(xb)
            assert torch.equal(oa, ob)
            oa.sum().backward()
            ob.sum().backward()
            assert torch.equal(xa.grad, xb.grad)
    assert sum("not covered by the kernels" in str(m.message) and "63 pixels" in str(m.message) for m in caught) == 1
    for a, b in zip(ours.state_dict().values(), ref.state_dict().values()):
        assert torch.equal(a, b)
    for a, b in zip(ours.parameters(), ref.parameters()):
        assert torch.equal(a.grad, b.grad)


def test_sgd_steps_b1_update_and_load_state_dict():
    # after each in-place update the swapped head computes what a fresh swap of the same parameters (a new pack) computes, bit for bit,
    # so the pack cache follows W1 and b1 each; the b1-only update must change the output
    ref = _head(24, 2, seed=2)
    ours = dec.FusedOutputHead.from_module(ref)
    opt = torch.optim.SGD(ours.parameters(), lr=0.05)
    x = torch.randn(3, 24, 9, 20, device="cuda")

    def fresh_eval():
        f = dec.FusedOutputHead.from_module(copy.deepcopy(ref)).eval()
        ours.eval()
        with _deterministic():
            want, got = f(x), ours(x)
        ours.train()
        assert torch.equal(got, want)
        return got

    for _ in range(3):
        opt.zero_grad()
        with _deterministic():
            (ours(x) * x[:, :2].cos()).sum().backward()
        opt.step()
        fresh_eval()
    assert int(ours[1].num_batches_tracked) == 3
    before = fresh_eval()
    with torch.no_grad():
        ours[3].bias.add_(0.25)
    after = fresh_eval()
    assert not torch.equal(before, after)
    ours.load_state_dict(_head(24, 2, seed=5).state_dict())
    fresh_eval()


# 6: y past 2^31 bytes in training
def test_training_past_2_31_bytes():
    maps, c, n, h, w = 19, 128, 2, 480, 480
    big = maps * c * h * w * 4
    assert big > 2 ** 31
    # y and grad_y, then the per-map fp64 restatement's temporaries (~10 of 236 MB)
    need = 2 * big + (6 << 30)
    free, _ = torch.cuda.mem_get_info()
    print(f"\nfree device memory {free / 2 ** 30:.1f} GiB, the test needs {need / 2 ** 30:.1f} GiB")
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    _, w1, b1, norm = oc.operands(1, c, n, 4, 4, seed=19)
    gen = torch.Generator(device="cuda").manual_seed(5)
    y = torch.randn(maps, c, h, w, device="cuda", generator=gen).mul_(0.5).add_(0.1)
    (out, mean, var), bufs = oc.fused_forward(y, w1, b1, norm, True)
    assert all(oc.margins_intact(b) for b in bufs)
    # the statistics against fp64 sums over two maps at a time
    cnt = maps * h * w
    chunks = lambda f: sum(f(y[j:j + 2].double()) for j in range(0, maps, 2))              # noqa: E731
    mu = chunks(lambda t: t.sum((0, 2, 3))) / cnt
    v64 = chunks(lambda t: ((t - mu.view(1, -1, 1, 1)) ** 2).sum((0, 2, 3))) / cnt
    sa = chunks(lambda t: t.abs().sum((0, 2, 3))) / cnt
    sd = chunks(lambda t: (t - mu.view(1, -1, 1, 1)).abs().sum((0, 2, 3))) / cnt
    em = oc.BN_SUM * oc.SUM * sa
    r = {"mean": gc.excess(mean, mu, em), "var": gc.excess(var, v64, 2 * oc.BN_SUM * oc.SUM * v64 + 4 * em * sd + em ** 2)}
    _note(r, "large_")
    _assert_within(r, "statistics")
    for j in (0, maps - 1):
        sl = slice(j, j + 1)
        st, _ = oc.stage_ratios((out[sl], mean, var), y[sl], w1, b1, norm, True, EPS)
        st = {"out": st["out"]}
        _note(st, "large_")
        _assert_within(st, ("out", j))
    del out, bufs
    # the backward: the parameter gradients against the sums of the per-map adjoints, grad_y of the first and last map from the whole
    # batch's totals
    g = torch.randn(maps, n, h, w, device="cuda", generator=gen)
    grads, gbufs = oc.fused_backward(g, y, mean, var, w1, b1, norm, True)
    assert all(oc.margins_intact(b) for b in gbufs)
    totals, want, bound = oc.batch_totals(y, g, w1, b1, norm, mean, var, True, EPS)
    r = {k: gc.excess(grads[oc.GRAD_KEYS.index(k)].reshape(want[k].shape), want[k], bound[k]) for k in ("gbw", "gbb", "gW", "gb")}
    nd = [t.double() for t in norm]
    for j in (0, maps - 1):
        sl = slice(j, j + 1)
        fj = oc.forward(y[sl].double(), w1, b1, nd, True, EPS, True, (mean.double(), var.double()))
        gj, bj = oc.adjoint(fj, w1, b1, nd, g[sl].double(), True, EPS, totals=totals, maps_total=maps)
        r[f"gy{j}"] = gc.excess(grads[0][sl], gj["gy"], bj["gy"])
    _note(r, "large_d_")
    _assert_within(r, "gradients")
