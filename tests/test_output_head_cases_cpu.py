"""The output head's fp64 restatement (tests/_output_head_cases.py) on the CPU: it equals the oracle head's own math without rounding,
its bounds hold for an fp32 evaluation in another order, and each planted defect is caught far outside them."""
from __future__ import annotations

import pytest
import torch

from oracle import decoder_oracle as DO
from tests import _output_head_cases as oc
from tests import _spatial_gru_cases as gc


def _oracle_head(c, n, norm, w1, b1, training):
    head = DO.output_head(c, n).double().train(training)
    with torch.no_grad():
        head[1].weight.copy_(norm[0]), head[1].bias.copy_(norm[1])
        head[1].running_mean.copy_(norm[2]), head[1].running_var.copy_(norm[3])
        head[3].weight.copy_(w1), head[3].bias.copy_(b1)
    return head


@pytest.mark.parametrize("training", [True, False])
def test_restatement_equals_oracle_head_without_rounding(training):
    maps, c, n, h, w = 2, 12, 3, 4, 8
    y, w1, b1, norm = oc.integer_operands(maps, c, n, h, w, device="cpu")
    y, w1, b1, norm = y.double(), w1.double(), b1.double(), [t.double() for t in norm]
    head = _oracle_head(c, n, norm, w1, b1, training)
    yr = y.clone().requires_grad_(True)
    want = head[3](head[2](head[1](yr)))
    g = torch.randint(-3, 4, want.shape, generator=torch.Generator().manual_seed(2)).double()
    want.backward(g)
    fw = oc.forward(y, w1, b1, norm, training, head[1].eps, rounding=False)
    grads, _ = oc.adjoint(fw, w1, b1, norm, g, training, head[1].eps)
    # the same formulas in fp64; only the order of a few fp64 operations differs (torch's batch norm vs the restatement's)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)       # noqa: E731
    close(fw["value"]["out"], want)
    for k, got in (("gy", yr.grad), ("gbw", head[1].weight.grad), ("gbb", head[1].bias.grad), ("gW", head[3].weight.grad.view(n, c))):
        close(grads[k], got)
    assert torch.equal(grads["gb"], head[3].bias.grad)


def _case(training, seed=0):
    maps, c, n, h, w = 3, 20, 2, 8, 12
    y, w1, b1, norm = oc.operands(maps, c, n, h, w, seed, device="cpu")
    g = torch.randn((maps, n, h, w), generator=torch.Generator().manual_seed(seed + 1))
    return y, w1, b1, norm, g


@pytest.mark.parametrize("training", [True, False])
def test_bounds_hold_for_fp32_in_another_order(training):
    y, w1, b1, norm, g = _case(training)
    fw64 = oc.forward(y.double(), w1, b1, [t.double() for t in norm], training, 1e-5)
    stats = (fw64["value"]["mean"].float(), fw64["value"]["var"].float())
    fw32 = oc.forward(y, w1, b1, norm, training, 1e-5, kernel=stats)       # fp32 sums in torch's order, not the kernels'
    run = (fw32["value"]["out"], stats[0], stats[1])
    ratios, fw = oc.stage_ratios(run, y, w1, b1, norm, training, 1e-5)
    assert all(same and r <= 1.0 for r, same in ratios.values()), ratios
    g32, _ = oc.adjoint(fw32, w1, b1, norm, g, training, 1e-5)
    got = [g32[k] for k in oc.GRAD_KEYS]
    r = oc.grad_ratios(fw, got, w1, b1, norm, g, training, 1e-5)
    assert all(same and v <= 1.0 for v, same in r.values()), r


# (training, eps) per defect where it is not (True, 1e-5): the batch statistics in eval need eval; with y's variance near 1/4 the two
# placements of eps agree to first order in eps, so that defect is shown in eval (running var near 1.1) at eps 1e-3
DEFECT_MODE = {"batch_stats_in_eval": (False, 1e-5), "eps_outside_sqrt": (False, 1e-3)}


@pytest.mark.parametrize("defect", sorted(oc.DEFECTS))
def test_planted_defects_caught(defect):
    training, eps = DEFECT_MODE.get(defect, (True, 1e-5))
    y, w1, b1, norm, g = _case(training, seed=3)
    nd = [t.double() for t in norm]
    clean = oc.forward(y.double(), w1, b1, nd, training, eps)
    bad = oc.forward(y.double(), w1, b1, nd, training, eps, defect=defect)
    ratios = [gc.excess(bad["value"][k], clean["value"][k], clean["bound"][k])[0] for k in ("out", "mean", "var")]
    want, bound = oc.adjoint(clean, w1, b1, nd, g.double(), training, eps)
    got, _ = oc.adjoint(bad if defect in oc.FORWARD_DEFECTS else clean, w1, b1, nd, g.double(), training, eps, defect=defect)
    ratios += [gc.excess(got[k], want[k], bound[k])[0] for k in oc.GRAD_KEYS]
    assert max(ratios) > 10, (defect, ratios)


@pytest.mark.parametrize("momentum", [0.1, None], ids=["momentum", "cumulative"])
@pytest.mark.parametrize("defect", [None] + sorted(oc.MODULE_DEFECTS))
def test_running_update_is_torchs(defect, momentum):
    # the module tests hold the running statistics to running_update: it is torch's own update of nn.BatchNorm2d within its bound, and
    # the biased-variance defect lands far outside it
    c, count = 6, 2 * 5 * 6
    bn = torch.nn.BatchNorm2d(c, momentum=momentum).double()
    x = torch.randn(2, c, 5, 6, generator=torch.Generator().manual_seed(4), dtype=torch.float64) * 0.7 + 0.2
    with torch.no_grad():
        bn.running_mean.uniform_(-0.5, 0.5), bn.running_var.uniform_(0.5, 1.5)
        bn.num_batches_tracked.fill_(2)
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    bn.train()(x)
    (wm, bm), (wv, bv) = oc.running_update(rm, rv, x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=False), count, momentum,
                                            int(bn.num_batches_tracked), defect)
    rm_ratio, _ = gc.excess(bn.running_mean, wm, bm)
    rv_ratio, _ = gc.excess(bn.running_var, wv, bv)
    if defect is None:
        assert rm_ratio <= 1.0 and rv_ratio <= 1.0, (rm_ratio, rv_ratio)
    else:
        assert rv_ratio > 10, rv_ratio


def test_batch_totals_give_the_whole_batch_adjoint():
    # the chunked adjoint of a batch too large to restate at once: its parameter gradients and the training dy of any one map from the
    # whole batch's totals are the whole-batch adjoint's
    training, eps = True, 1e-5
    y, w1, b1, norm, g = _case(training, seed=5)
    nd = [t.double() for t in norm]
    fw = oc.forward(y.double(), w1, b1, nd, training, eps)
    mean, var = fw["value"]["mean"].float(), fw["value"]["var"].float()
    fw = oc.forward(y.double(), w1, b1, nd, training, eps, True, (mean.double(), var.double()))
    want, bound = oc.adjoint(fw, w1, b1, nd, g.double(), training, eps)
    totals, grads, bounds = oc.batch_totals(y, g, w1, b1, norm, mean, var, training, eps, chunk=1)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-14)       # noqa: E731
    for k in ("gbw", "gbb", "gW", "gb"):
        close(grads[k], want[k])
        close(bounds[k], bound[k])
    for j in range(y.shape[0]):
        fj = oc.forward(y[j:j + 1].double(), w1, b1, nd, training, eps, True, (mean.double(), var.double()))
        gj, bj = oc.adjoint(fj, w1, b1, nd, g[j:j + 1].double(), training, eps, totals=totals, maps_total=y.shape[0])
        close(gj["gy"], want["gy"][j:j + 1])
        close(bj["gy"], bound["gy"][j:j + 1])


@pytest.mark.parametrize("sms", [132, 114])
def test_envelope_reaches_every_launch_case(sms):
    # the host model of the forward's launch: the table reaches every K padding class with its ring depth, every n in two classes, each
    # last-tile split, each piece edge, the minimum count and a tile count off the grid; the wrap cases make every CTA use each ring
    # stage at least twice and change maps between its tiles, at every K padding class
    assert {k: oc.ring_depth(k) for k in oc.KPADS} == {32: 4, 64: 4, 96: 3, 128: 2}
    rs = [oc.reach(case, sms) for case in oc.ENVELOPE]
    assert {c for _, c, *_ in oc.ENVELOPE} >= {1, 2, 8, 31, 32, 33, 63, 64, 65, 96, 97, 127, 128}
    for n in range(1, 9):
        assert len({r["kpad"] for r in rs if r["n"] == n}) >= 2, n
    assert {r["tail"] for r in rs} >= {4, 60, 64, 68, 124, 0}
    assert {r["wg1_valid"] for r in rs if r["wg1_valid"] <= 0} >= {-60, -4, 0} and any(0 < r["wg1_valid"] < 64 for r in rs)
    assert {h * w for _, _, _, h, w, _ in oc.ENVELOPE} >= {4092, 4096, 4100, 8188}
    assert any(r["min_count"] for r in rs)
    assert any(r["uneven"] and r["min_per_cta"] < 2 for r in rs)
    assert {t for *_, t in oc.ENVELOPE} == {True, False} and len(oc.ENVELOPE) == 2 * len(oc.SHAPES)
    for kp in oc.KPADS:
        case = oc.wrap_case(kp, sms)
        r = oc.reach(case, sms)
        assert r["kpad"] == kp and r["ring_wrap"] and r["frame_change"] and r["wg1_valid"] > 0, (kp, r)
        assert not oc.reach((case[0] - 1,) + case[1:], sms)["ring_wrap"]
    for case in oc.SHIPPED:
        r = oc.reach(case, sms)
        assert r["wg1_valid"] == 0 and r["tiles"] == case[0] * 313 and r["ring_wrap"]
