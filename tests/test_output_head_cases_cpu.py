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


@pytest.mark.parametrize("defect", sorted(oc.DEFECTS))
def test_planted_defects_caught(defect):
    training = defect != "batch_stats_in_eval"
    y, w1, b1, norm, g = _case(training, seed=3)
    nd = [t.double() for t in norm]
    clean = oc.forward(y.double(), w1, b1, nd, training, 1e-5)
    bad = oc.forward(y.double(), w1, b1, nd, training, 1e-5, defect=defect)
    ratios = [gc.excess(bad["value"][k], clean["value"][k], clean["bound"][k])[0] for k in ("out", "mean", "var")]
    want, bound = oc.adjoint(clean, w1, b1, nd, g.double(), training, 1e-5)
    got, _ = oc.adjoint(bad if defect in ("w1_transposed", "unbiased_var", "batch_stats_in_eval") else clean, w1, b1, nd, g.double(),
                        training, 1e-5, defect=defect)
    ratios += [gc.excess(got[k], want[k], bound[k])[0] for k in oc.GRAD_KEYS]
    assert max(ratios) > 10, (defect, ratios)
