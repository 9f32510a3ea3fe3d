"""CPU: the Bottleneck restatement of tests/_bottleneck_cases.py against the fp64 oracle module, its element-wise bounds against an fp32
evaluation in another summation order (sound) and against kernels with planted defects (not vacuous), and the envelope table against
the C ABI's launch rules and limits."""
from __future__ import annotations

import pytest
import torch

from fiery_b200 import _lib
from fiery_b200 import bottleneck as bk
from oracle.future_oracle import Bottleneck
from tests import _bottleneck_cases as bc

EPS = 1e-5


def _case(maps, c, h, w, seed=0, dtype=torch.float64):
    """operands() on the host: fp32 values held in ``dtype``, and an output gradient"""
    x, weights, norms = bc.operands(maps, c, h, w, seed=seed, device="cpu")
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(seed + 1))
    return x.to(dtype), [t.to(dtype) for t in weights], [t.to(dtype) for t in norms], g.to(dtype)


def _oracle(c, weights, norms, training):
    b = Bottleneck(c).double().train(training)
    bns = [b.layers.abn_down_project[0], b.layers.abn[0], b.layers.abn_up_project[0]]
    with torch.no_grad():
        for conv, wt in zip((b.layers.conv_down_project, b.layers.conv, b.layers.conv_up_project), weights):
            conv.weight.copy_(wt)
        for i, bn in enumerate(bns):
            for j, name in enumerate(("weight", "bias", "running_mean", "running_var")):
                getattr(bn, name).copy_(norms[4 * i + j])
            bn.eps = EPS
    return b


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("shape", [(2, 17, 7, 8), (1, 6, 5, 4), (3, 10, 9, 12)], ids=lambda s: "x".join(map(str, s)))
def test_restatement_matches_the_oracle(shape, training):
    x, weights, norms, g = _case(*shape, seed=sum(shape))
    m = _oracle(shape[1], weights, norms, training)
    xr = x.clone().requires_grad_(True)
    out = m(xr)
    out.backward(g)
    fw = bc.forward(x, weights, norms, training, EPS, rounding=False)
    assert float((fw["value"]["out"] - out.detach()).abs().max()) < 1e-12
    grads, _ = bc.adjoint(fw, weights, norms, g, training, EPS)
    bns = [m.layers.abn_down_project[0], m.layers.abn[0], m.layers.abn_up_project[0]]
    want = {"dx": xr.grad, "gW_down": m.layers.conv_down_project.weight.grad, "gW_conv": m.layers.conv.weight.grad,
            "gW_up": m.layers.conv_up_project.weight.grad}
    for i, bn in enumerate(bns):
        want[f"gw{i + 1}"], want[f"gb{i + 1}"] = bn.weight.grad, bn.bias.grad
    for k, wv in want.items():
        assert float((grads[k] - wv).abs().max()) < 1e-12 * max(float(wv.abs().max()), 1.0), k


def _fp32_run(x, weights, norms, g, training, defect=None):
    """the restatement evaluated in fp32 (its own matmul and reduction orders; a planted defect optional), as a run the checks take"""
    f = lambda ts: [t.float() if t is not None else None for t in ts]      # noqa: E731
    fw = bc.forward(x.float(), f(weights), f(norms), training, EPS, rounding=True, defect=defect)
    v = fw["value"]
    run = bc.as_run(v["out"], v["y1"], v["y2"], v["y3"], torch.cat([v[k] for k in ("mean1", "var1", "mean2", "var2", "mean3", "var3")]))
    grads, _ = bc.adjoint(fw, f(weights), f(norms), g.float(), training, EPS, defect=defect)
    return run, [grads[k] for k in bc.GRAD_KEYS]


SOUND = [(2, 17, 7, 8), (3, 2, 1, 4), (1, 66, 9, 20), (4, 35, 8, 36), (300, 16, 1, 4)]


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("shape", SOUND, ids=lambda s: "x".join(map(str, s)))
def test_bounds_are_sound(shape, training):
    x, weights, norms, g = _case(*shape, seed=3 + shape[1])
    run, grads = _fp32_run(x, weights, norms, g, training)
    stages, fw = bc.stage_ratios(run, x, weights, norms, training, EPS)
    for st, (ratio, same) in stages.items():
        assert same and ratio <= 1.0, (st, ratio)
    ratios = bc.grad_ratios(fw, grads, weights, norms, g, training, EPS)
    assert set(ratios) == set(bc.GRAD_KEYS)
    for k, (ratio, same) in ratios.items():
        assert same and ratio <= 1.0, (k, ratio)
    # the fp32 run is not the restatement: its sums run in another order (one-term sums at M = 1 are exact either way)
    assert shape[1] < 4 or float((run["y2"].double() - fw["value"]["y2"]).abs().max()) > 0


@pytest.mark.parametrize("defect", list(bc.DEFECTS))
def test_bounds_are_not_vacuous(defect):
    shape = (1, 24, 2, 32)                                       # two 32-pixel runs, every pixel on the map's edge
    x, weights, norms, g = _case(*shape, seed=5)
    norms[1] = norms[1].abs() + 2.0                                # bn1's shift > 0, so the prologue would fill with relu(shift) > 0
    training = defect == "unbiased_var"                          # eval elsewhere: the tighter bounds of an eval norm's backward
    run, grads = _fp32_run(x, weights, norms, g, training, defect)
    stages, fw = bc.stage_ratios(run, x, weights, norms, training, EPS)
    worst = max(r if same else float("inf") for r, same in stages.values())
    if defect in ("run_dropped", "wgrad_halo"):
        worst = max(r for r, _ in bc.grad_ratios(fw, grads, weights, norms, g, training, EPS).values())
    print(f"{defect}: largest err/bound {worst:.3g}")
    assert worst > 10, (defect, stages)


def test_unfold_convolutions_keep_a_nan_where_a_direct_convolution_puts_it():
    x = torch.randn(2, 3, 6, 8, dtype=torch.float64)
    w = torch.randn(4, 3, 1, 1, dtype=torch.float64)
    x[1, 2, 5, 0] = float("nan")
    want = torch.zeros(2, 4, 6, 8, dtype=torch.bool)
    want[1, :, 5, 0] = True
    assert torch.equal(torch.isnan(bc._mm(w, x)), want)
    assert torch.allclose(bc._mm(w, x.nan_to_num()), torch.nn.functional.conv2d(x.nan_to_num(), w))


def test_fmaf_is_rounded_once():
    # 1 + 2^-24 + 2^-60: the fp64 sum rounds to the midpoint 1 + 2^-24 and then to 1 (ties to even); the fma rounds up
    a = torch.tensor([1.0 + 2 ** -23], dtype=torch.float64)
    y = torch.tensor([2 ** -30 + 2 ** -53], dtype=torch.float64).float().double()
    c = torch.tensor([1.0], dtype=torch.float64)
    exact = bc.fmaf_exact(a.numpy(), y.numpy(), c.numpy())
    assert float(bc.fmaf(a, y, c)[0]) == float(exact[0])
    r = torch.randn(1000, dtype=torch.float64).float().double()
    s, sh = torch.randn(1000).double(), torch.randn(1000).double()
    assert torch.equal(bc.fmaf(s, r, sh), torch.from_numpy(bc.fmaf_exact(s.numpy(), r.numpy(), sh.numpy())).double())


def test_envelope_reaches_every_instantiation_and_its_edges_are_rejected():
    lib = _lib.load()
    reached = set()
    for maps, c, h, w in bc.ENVELOPE:
        assert all(v > 0 for v in bk.workspace_bytes(maps, h, w, c)), (maps, c, h, w)
        reached |= bc.instantiations(maps, c, h, w)
    want = {(k, n) for k in ("bottleneck_conv_fwd_kernel", "bottleneck_conv_wgrad_kernel") for n in range(8, 65, 8)}
    want |= {(k, n) for k in ("bottleneck_entry_fwd_kernel", "bottleneck_entry_dgrad_kernel") for n in (1, 2)}
    want |= {("bottleneck_entry_wgrad_kernel", 1)}
    assert reached == want
    ms = {c // 2 for _, c, _, _ in bc.ENVELOPE}
    assert {1, 9, 16, 41, 48, 49, 56, 64} <= ms                        # both ends of the widths
    cs = {c for _, c, _, _ in bc.ENVELOPE}
    assert {2, 128} <= cs and any(c % 2 for c in cs)
    assert {1, 7, 8, 9, 17} <= {s[2] for s in bc.ENVELOPE}
    assert {4, 12, 16, 20, 32, 36, 132} <= {s[3] for s in bc.ENVELOPE}
    assert {4096, 4160} <= {s[2] * s[3] for s in bc.ENVELOPE} and any(s[2] * s[3] < 32 for s in bc.ENVELOPE)
    tiles = [bc.wgrad_tiles(maps, h, w) for maps, _, h, w in bc.ENVELOPE]
    assert any(t3 > bc.WG_MAX_CHUNKS and t3 % bc.WG_MAX_CHUNKS for t3, _ in tiles)
    assert any(t1 > bc.WG_MAX_CHUNKS and t1 % bc.WG_MAX_CHUNKS for _, t1 in tiles)
    assert (12, 64, 200, 200) in bc.ENVELOPE
    for field, value, msg in [("channels", 1, "channels = 1"), ("channels", 129, "channels = 129"), ("grid_y", 0, "grid_y = 0"),
                              ("grid_y", 6, "grid_y = 6"), ("eps", -1e-3, "eps = "), ("training", 2, "training = 2")]:
        d = bk.desc(2, 8, 8, 64)
        setattr(d, field, value)
        assert lib.fiery_bottleneck_forward_workspace_bytes(d) == 0 and lib.fiery_bottleneck_backward_workspace_bytes(d) == 0
        assert lib.fiery_bottleneck_forward(d, *([None] * 10)) != 0 and msg in lib.fiery_last_error().decode(), msg
    d = bk.desc(1, 1 << 16, 1 << 15, 64)                                 # X * Y = 2^31 pixels
    assert lib.fiery_bottleneck_forward_workspace_bytes(d) == 0
    assert lib.fiery_bottleneck_forward(d, *([None] * 10)) != 0
    assert lib.fiery_last_error().decode()

