"""CPU: the SpatialGRU restatement of tests/_spatial_gru_cases.py against the fp64 oracle module, its element-wise bounds against an
fp32 evaluation in another summation order (sound) and against wrong parameters (not vacuous), TF32 rounding's three modes on their
ties, and the shape list against the C ABI's limits."""
from __future__ import annotations

import copy

import pytest
import torch

from tests import _spatial_gru_cases as gc
from fiery_b200 import _lib
from fiery_b200.future_prediction import _desc, workspace_bytes
from oracle.future_oracle import SpatialGRU


def _oracle(cx, ch, p, bias_init, training, eps=1e-5):
    m = SpatialGRU(cx, ch, gru_bias_init=bias_init).double().train(training)
    with torch.no_grad():
        m.conv_update.weight.copy_(p["w_gates"][:ch])
        m.conv_reset.weight.copy_(p["w_gates"][ch:])
        m.conv_update.bias.copy_(p["b_gates"][:ch])
        m.conv_reset.bias.copy_(p["b_gates"][ch:])
        m.conv_state_tilde.conv.weight.copy_(p["w_state"])
        bn = m.conv_state_tilde.norm
        bn.weight.copy_(p["gamma"])
        bn.bias.copy_(p["beta"])
        bn.running_mean.copy_(p["running_mean"])
        bn.running_var.copy_(p["running_var"])
        bn.eps = eps
    return m


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("case", [(5, 6, 7, 8, 2, 3, 3, 0.0), (3, 9, 5, 4, 3, 2, 1, 0.75), (8, 4, 9, 12, 1, 1, 1, -0.5)],
                         ids=gc.case_id)
def test_restatement_matches_the_oracle(case, training):
    cx, ch, X, Y, b, T, Tx, bias_init = case
    p = gc.params(cx, ch, seed=cx + ch)
    x, h0, go = gc.inputs(b, T, Tx, cx, ch, X, Y, seed=3)
    m = _oracle(cx, ch, p, bias_init, training)
    xr = x.expand(b, T, cx, X, Y).clone().requires_grad_(True) if Tx == 1 else x.clone().requires_grad_(True)
    hr = h0.clone().requires_grad_(True)
    out = m(xr, hr)
    out.backward(go)
    fw = gc.forward(x, h0, p, T, training, 1e-5, bias_init, rounding=False)
    got = torch.stack(fw["value"]["out"], 1)
    assert (got - out.detach()).abs().max() < 1e-13
    grads, _ = gc.adjoint(fw, x, h0, p, go, training, 1e-5)
    gx = xr.grad.sum(1, keepdim=True) if Tx == 1 else xr.grad
    want = {"x": gx, "h0": hr.grad, "w_gates": torch.cat([m.conv_update.weight.grad, m.conv_reset.weight.grad]),
            "b_gates": torch.cat([m.conv_update.bias.grad, m.conv_reset.bias.grad]), "w_state": m.conv_state_tilde.conv.weight.grad,
            "gamma": m.conv_state_tilde.norm.weight.grad, "beta": m.conv_state_tilde.norm.bias.grad}
    for k, w in want.items():
        scale = max(float(w.abs().max()), 1.0)
        assert float((grads[k] - w).abs().max()) < 1e-13 * scale, k


def _fp32_run(x, h0, p, T, training, bias_init, go):
    """the restatement evaluated in fp32 on the CPU (its own matmul and reduction orders), as a run the checks take"""
    p32 = {k: (v.float() if v is not None else None) for k, v in p.items()}
    fw = gc.forward(x.float(), h0.float(), p32, T, training, 1e-5, bias_init, rounding=True)
    v = fw["value"]
    run = {"out": torch.stack(v["out"], 1), "u": torch.stack(v["u"]), "r": torch.stack(v["r"]), "q": torch.stack(v["q"]),
           "s": torch.stack(v["s"]), "means": torch.stack(v["mean"]), "vars": torch.stack(v["var"])}
    grads, _ = gc.adjoint(fw, x.float(), h0.float(), p32, go.float(), training, 1e-5)
    return run, grads


SOUND = [(5, 6, 7, 8, 2, 3, 3, 0.0), (9, 33, 9, 20, 3, 2, 1, 0.75), (64, 64, 8, 16, 1, 2, 2, -0.5), (1, 1, 1, 4, 3, 2, 1, 0.0)]


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("case", SOUND, ids=gc.case_id)
def test_bounds_are_sound(case, training):
    cx, ch, X, Y, b, T, Tx, bias_init = case
    p = gc.params(cx, ch, seed=11 + cx)
    x, h0, go = gc.inputs(b, T, Tx, cx, ch, X, Y, seed=5)
    x, h0, go = x.float().double(), h0.float().double(), go.float().double()
    run, grads = _fp32_run(x, h0, p, T, training, bias_init, go)
    stages, fw = gc.stage_ratios(run, x, h0, p, T, training, 1e-5, bias_init)
    for st, (ratio, same) in stages.items():
        assert same and ratio <= 1.0, (st, ratio)
    for k, (ratio, same) in gc.grad_ratios(fw, grads, x, h0, p, go, training, 1e-5).items():
        assert same and ratio <= 1.0, (k, ratio)


@pytest.mark.parametrize("wrong", ["tap", "bias", "bias_init", "state_tap"])
def test_bounds_are_not_vacuous(wrong):
    cx, ch, X, Y, b, T, bias_init = 6, 8, 7, 8, 2, 2, 0.75
    p = gc.params(cx, ch, seed=4)
    x, h0, go = gc.inputs(b, T, T, cx, ch, X, Y, seed=6)
    bad = copy.deepcopy(p)
    bad_init = bias_init
    if wrong == "tap":
        bad["w_gates"][ch + 2, cx + 1, 0, 2] += 0.25          # the r gate, an h input, one tap
    elif wrong == "bias":
        bad["b_gates"][3] = 0.0
    elif wrong == "bias_init":
        bad_init = 0.0
    else:
        bad["w_state"][1, 0, 1, 1] += 0.25
    run, grads = _fp32_run(x, h0, bad, T, True, bad_init, go)
    stages, fw = gc.stage_ratios(run, x, h0, p, T, True, 1e-5, bias_init)
    first = {"tap": "r", "bias": "u", "bias_init": "u", "state_tap": "s"}[wrong]
    assert stages[first][0] > 10, stages
    # a wrong weight also leaves the gradients outside the right model's adjoint (the biases reach the adjoint only through the saved
    # gates, which it takes from the run)
    if wrong in ("tap", "state_tap"):
        ratios = gc.grad_ratios(fw, grads, x, h0, p, go, True, 1e-5)
        assert max(ratios["x"][0], ratios["h0"][0]) > 1, ratios


def test_tf32_modes_on_their_ties():
    v = torch.tensor([1 + 2 ** -11, 1 + 2 ** -12, 1 - 2 ** -12, 1 + 3 * 2 ** -12, -(1 + 2 ** -11), 1 + 3 * 2 ** -11], dtype=torch.float64)
    assert gc.tf32_rna(v).tolist() == [1 + 2 ** -10, 1, 1, 1 + 2 ** -10, -(1 + 2 ** -10), 1 + 2 ** -9]
    assert gc.tf32_rne(v).tolist() == [1, 1, 1, 1 + 2 ** -10, -1, 1 + 2 ** -9]
    assert gc.tf32_rz(v).tolist() == [1, 1, 1 - 2 ** -11, 1, -1, 1 + 2 ** -10]
    # a NaN with a full payload (the GPU's 0x7fffffff) stays NaN: the rounding bias must not carry into the sign bit
    full = torch.tensor([0x7FFFFFFF, -1], dtype=torch.int32).view(torch.float32)
    for f in (gc.tf32_rna, gc.tf32_rz, gc.tf32_rne):
        assert bool(torch.isnan(f(full)).all()) and bool(torch.isnan(f(full.double())).all())
    special = torch.tensor([float("inf"), float("-inf"), float("nan"), 0.0, -0.0])
    for f in (gc.tf32_rna, gc.tf32_rz, gc.tf32_rne):
        r = f(special)
        assert r[0] == float("inf") and r[1] == float("-inf") and torch.isnan(r[2]) and r[3] == 0 and r[4] == 0


def test_unfold_convolutions_match_torch_and_keep_nan_where_a_direct_convolution_puts_it():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 5, 7, 8, generator=g, dtype=torch.float64)
    w = torch.randn(3, 5, 3, 3, generator=g, dtype=torch.float64)
    gy = torch.randn(2, 3, 7, 8, generator=g, dtype=torch.float64)
    F = torch.nn.functional
    assert torch.allclose(gc.conv(x, w), F.conv2d(x, w, padding=1), atol=1e-12)
    assert torch.allclose(gc.conv_t(gy, w), torch.nn.grad.conv2d_input(x.shape, w, gy, padding=1), atol=1e-12)
    assert torch.allclose(gc.conv_w(x, gy), torch.nn.grad.conv2d_weight(x, w.shape, gy, padding=1), atol=1e-12)
    x[1, 2, 0, 7] = float("nan")
    y = gc.conv(x, w)
    want = torch.zeros(2, 3, 7, 8, dtype=torch.bool)
    want[1, :, 0:2, 6:8] = True
    assert torch.equal(torch.isnan(y), want)


def test_shape_list_is_inside_the_abi_and_its_edges_are_outside():
    seen_cx, seen_ch, ns = set(), set(), set()
    for cx, ch, X, Y, b, T, Tx, _ in gc.CASES:
        assert all(v > 0 for v in workspace_bytes(b, T, Tx, X, Y, cx, ch)), (cx, ch, X, Y, b, T, Tx)
        seen_cx.add(cx)
        seen_ch.add(ch)
        rows = (2 * ch + 7) // 8 * 8                             # the gates' N = round8(2 C_h), then the instantiated width
        ns.add(rows if rows <= 64 else (96 if rows <= 96 else 128))
    assert set(gc.CHANNELS) <= seen_cx and set(gc.CHANNELS) <= seen_ch
    assert ns == {8, 16, 24, 32, 40, 48, 56, 64, 96, 128}      # every instantiation of the gates' convolution
    assert any(33 <= ch <= 60 for ch in seen_ch)
    assert {1, 7, 8, 9, 200} <= {c[2] for c in gc.CASES} and {4, 12, 16, 20, 200} <= {c[3] for c in gc.CASES}
    assert {1, 3} <= {c[4] for c in gc.CASES} and {1, 2, 5} <= {c[5] for c in gc.CASES}
    assert any(c[6] == 1 and c[5] > 1 for c in gc.CASES) and any(c[6] == c[5] > 1 for c in gc.CASES)
    lib = _lib.load()
    for args, msg in [((1, 2, 1, 4, 8, 0, 8), b"x_channels = 0"), ((1, 2, 1, 4, 8, 65, 8), b"x_channels = 65"),
                      ((1, 2, 1, 4, 8, 8, 0), b"h_channels = 0"), ((1, 2, 1, 4, 8, 8, 65), b"h_channels = 65"),
                      ((1, 2, 1, 4, 6, 8, 8), b"grid_y = 6"), ((1, 3, 2, 4, 8, 8, 8), b"x_frames = 2")]:
        d = _desc(*args)
        assert lib.fiery_spatial_gru_saved_bytes(d) == 0 and lib.fiery_spatial_gru_backward_workspace_bytes(d) == 0
        assert lib.fiery_spatial_gru_forward(d, *([None] * 14)) == -1 and msg in lib.fiery_last_error(), msg


def test_input_rule_copies_a_misaligned_fp32_map():
    from fiery_b200.future_prediction import gru_input
    buf = torch.zeros(2 * 3 * 4 * 5 * 8 + 1)
    x = buf[1:].view(2, 3, 4, 5, 8)
    assert x.is_contiguous() and x.data_ptr() % 16 != 0
    y = gru_input(x)
    assert y is not x and y.data_ptr() % 16 == 0 and torch.equal(y, x)
    z = torch.zeros(2, 3, 4, 5, 8)
    assert gru_input(z) is z
    s0 = torch.zeros(1, 3, 4, 5, 8).expand(2, 3, 4, 5, 8)      # a stride-0 batch is read in place
    assert gru_input(s0) is s0
