"""CPU: the SpatialGRU swap's coverage rules and warnings on oracle models, the operator's fakes against the C ABI's sizes, the
kernels' input rule (a stride-0 time dimension stays one frame, a broadcast map is materialized once), and the C ABI's limits."""
from __future__ import annotations

import copy
import warnings

import pytest
import torch
import torch.nn as nn
from torch.fx.experimental.proxy_tensor import make_fx

from fiery_b200 import _lib, install
from fiery_b200.future_prediction import TensorCoreSpatialGRU, gru_input, module_reason, unsupported_reason, workspace_bytes
from oracle.future_oracle import FuturePrediction, SpatialGRU


class Holder(nn.Module):
    def __init__(self, fp=None):
        super().__init__()
        if fp is not None:
            self.future_prediction = fp


def _fresh_warnings():
    install._warned.clear()


def test_covered_and_uncovered_modules():
    assert module_reason(SpatialGRU(32, 64)) is None
    assert module_reason(SpatialGRU(64, 64)) is None
    assert "hidden_size = 65" in module_reason(SpatialGRU(32, 65))
    assert "input_size = 96" in module_reason(SpatialGRU(96, 64))
    g = SpatialGRU(8, 8)
    g.conv_update = nn.Conv2d(16, 8, 5, padding=2)
    assert "3x3" in module_reason(g)
    g = SpatialGRU(8, 8)
    g.conv_state_tilde.norm = nn.SyncBatchNorm(8)
    assert "SyncBatchNorm" in module_reason(g)
    g = SpatialGRU(8, 8)
    g.conv_state_tilde.activation = nn.Tanh()
    assert "Tanh" in module_reason(g)
    assert "does not have" in module_reason(nn.Linear(2, 2))
    assert unsupported_reason(8, 8, 30) is not None and unsupported_reason(8, 8, 32) is None


def test_swap_keeps_keys_is_idempotent_and_leaves_models_without_future_prediction():
    _fresh_warnings()
    fp = FuturePrediction(64, 32)
    model = Holder(fp)
    keys = list(model.state_dict().keys())
    before = [id(p) for p in model.parameters()]
    assert install.use_tensor_core_future_prediction(model) is model
    grus = list(model.future_prediction.spatial_grus)
    assert all(isinstance(g, TensorCoreSpatialGRU) for g in grus)
    assert list(model.state_dict().keys()) == keys
    assert [id(p) for p in model.parameters()] == before          # the same Parameters
    install.use_tensor_core_future_prediction(model)
    assert list(model.future_prediction.spatial_grus) == grus       # a second call does nothing
    bare = Holder()
    assert install.use_tensor_core_future_prediction(bare) is bare


def test_uncovered_grus_stay_with_one_warning():
    _fresh_warnings()
    fp = FuturePrediction(64, 32)
    fp.spatial_grus[1].conv_state_tilde.norm = nn.SyncBatchNorm(64)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        install.use_tensor_core_future_prediction(Holder(fp))
        install.use_tensor_core_future_prediction(Holder(fp))
    msgs = [str(x.message) for x in w if "SpatialGRU" in str(x.message)]
    assert len(msgs) == 1 and "spatial_grus[1]" in msgs[0] and "SyncBatchNorm" in msgs[0]
    assert isinstance(fp.spatial_grus[0], TensorCoreSpatialGRU) and isinstance(fp.spatial_grus[2], TensorCoreSpatialGRU)
    assert type(fp.spatial_grus[1]) is SpatialGRU


def test_call_time_fallback_matches_the_reference_on_cpu():
    _fresh_warnings()
    torch.manual_seed(0)
    ref = SpatialGRU(4, 8).eval()
    ours = TensorCoreSpatialGRU.from_module(copy.deepcopy(ref))
    x, h0 = torch.randn(2, 3, 4, 5, 6), torch.randn(2, 8, 5, 6)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = ours(x, h0)
    assert torch.equal(out, ref(x, h0))
    assert any("CPU input" in str(m.message) for m in w)


def test_input_rule():
    x = torch.randn(2, 1, 32, 1, 1).expand(2, 4, 32, 8, 8)
    one = x[:, :1]
    kept = gru_input(one)
    assert kept.shape == (2, 1, 32, 8, 8) and kept.is_contiguous()       # the broadcast map materialized, one frame
    full = torch.randn(2, 4, 32, 8, 8)
    assert gru_input(full) is full
    assert gru_input(full[:, 1:3]) is not None and gru_input(full[:, 1:3]).data_ptr() == full[:, 1:3].data_ptr()
    assert gru_input(full.half()).dtype == torch.float32


def test_fakes_have_the_c_abi_sizes():
    import fiery_b200.future_prediction  # noqa: F401  (registers the operator)
    b, T, cx, ch, h, w = 3, 4, 32, 64, 8, 12
    gru = SpatialGRU(cx, ch)
    bn = gru.conv_state_tilde.norm
    x, h0 = torch.zeros(b, 1, cx, h, w), torch.zeros(b, ch, h, w)
    params = [t.detach() for t in (gru.conv_update.weight, gru.conv_update.bias, gru.conv_reset.weight, gru.conv_reset.bias,
                                   gru.conv_state_tilde.conv.weight, bn.weight, bn.bias)]

    def f(x, h0, wu, bu, wr, br, ws, bnw, bnb):
        return torch.ops.fiery_b200.spatial_gru(x, h0, wu, bu, wr, br, ws, bnw, bnb, None, None, T, True, bn.eps, 0.0)

    gm = make_fx(f, tracing_mode="fake")(x, h0, *params)
    (node,) = [n for n in gm.graph.nodes if n.op == "output"]
    out, means, var, saved = (v.meta["val"] for v in node.args[0])
    assert out.shape == (b, T, ch, h, w) and out.dtype == torch.float32
    assert means.shape == var.shape == (T, ch)
    assert saved.dtype == torch.uint8 and saved.numel() == workspace_bytes(b, T, 1, h, w, cx, ch)[1]

    def g(gout, x, h0, out, saved, means, var, wu, wr, ws, bnw, bnb):
        return torch.ops.fiery_b200.spatial_gru_backward(gout, x, h0, out, saved, means, var, wu, wr, ws, bnw, bnb, T, True, bn.eps,
                                                         0.0, True, False, True, True, True)

    gm = make_fx(g, tracing_mode="fake")(torch.zeros(b, T, ch, h, w), x, h0, torch.zeros(b, T, ch, h, w),
                                         torch.zeros(saved.numel(), dtype=torch.uint8), torch.zeros(T, ch), torch.zeros(T, ch),
                                         params[0], params[2], params[4], params[5], params[6])
    (node,) = [n for n in gm.graph.nodes if n.op == "output"]
    shapes = [tuple(v.meta["val"].shape) for v in node.args[0]]
    assert shapes == [(b, 1, cx, h, w), (0,), (ch, cx + ch, 3, 3), (ch,), (ch, cx + ch, 3, 3), (ch,), (ch, cx + ch, 3, 3), (ch,), (ch,)]


def test_workspace_sizes_and_limits():
    b, T, h, w = 3, 4, 200, 200
    pack, saved, fwd, bwd = workspace_bytes(b, T, 1, h, w, 32, 64)
    assert saved == 4 * 4 * T * b * 64 * h * w
    assert pack > 0 and fwd > 0
    # dG (2 C_h) and ds (C_h) of every step, da and the carried state gradient, at least
    assert bwd >= 4 * (3 * T + 2) * b * 64 * h * w
    assert workspace_bytes(b, T, T, h, w, 64, 64)[3] > bwd              # the weight-gradient partials grow with C_x
    for bad in ((b, T, 1, h, w, 65, 64), (b, T, 1, h, w, 32, 0), (b, T, 2, h, w, 32, 64), (b, T, 1, h, 202, 32, 64),
                (0, T, 1, h, w, 32, 64)):
        assert workspace_bytes(*bad) == (0, 0, 0, 0), bad


def test_invalid_descriptor_messages():
    from fiery_b200.future_prediction import _desc
    lib = _lib.load()
    d = _desc(1, 2, 1, 4, 6, 8, 8)
    rc = lib.fiery_spatial_gru_forward(d, *([None] * 13), None)
    assert rc == -1 and b"grid_y = 6" in lib.fiery_last_error()
    d = _desc(1, 2, 1, 4, 8, 8, 80)
    assert lib.fiery_spatial_gru_forward(d, *([None] * 14)) == -1 and b"h_channels = 80" in lib.fiery_last_error()
    d = _desc(1, 2, 1, 4, 8, 8, 8, (6, 8, 4))
    assert lib.fiery_spatial_gru_packed_bytes(d) == 0
    lib.fiery_spatial_gru_forward(d, *([None] * 14))
    assert b"multiples of 4" in lib.fiery_last_error()


@pytest.mark.parametrize("cx,ch", [(32, 64), (64, 64), (1, 8), (35, 29), (64, 1)])
def test_pack_sizes(cx, ch):
    pack = workspace_bytes(1, 1, 1, 1, 4, cx, ch)[0]
    assert pack > 0 and pack % 1024 == 0


def test_conv3x3_limits_and_workspace():
    from fiery_b200.future_prediction import conv3x3_desc
    lib = _lib.load()
    ok = conv3x3_desc(3, 200, 200, (32, 48), (48, 48))
    assert lib.fiery_conv3x3_packed_bytes(ok) > 0
    # chunks (min(tiles, 128)) x 9 taps x all outputs x all inputs
    assert lib.fiery_conv3x3_backward_weight_workspace_bytes(ok) == 128 * 9 * 96 * 80 * 4
    assert lib.fiery_conv3x3_packed_bytes(conv3x3_desc(1, 4, 8, (8, 0), (8, 0))) > 0
    for bad, msg in (((0, 4, 8, (8, 8), (8, 8)), b"maps = 0"), ((1, 4, 8, (0, 8), (8, 8)), b"in_channels[0] = 0"),
                     ((1, 4, 8, (8, 65), (8, 8)), b"in_channels[1] = 65"), ((1, 4, 8, (8, 8), (8, 80)), b"out_channels[1] = 80"),
                     ((1, 4, 6, (8, 8), (8, 8)), b"grid_y = 6")):
        assert lib.fiery_conv3x3_packed_bytes(conv3x3_desc(*bad)) == 0
        assert msg in lib.fiery_last_error(), msg
