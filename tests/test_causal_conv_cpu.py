"""CPU: the causal convolution's host side -- the C ABI's shape limits and workspace rule, the adopted module, the install helper on
TemporalBlock, TensorCoreTemporalBlock and Bottleneck3D (in either order with the temporal-block swap), and the operators' fakes under a
symbolic trace."""
import warnings

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.fx.experimental.proxy_tensor import make_fx
from torch.fx.experimental.symbolic_shapes import ShapeEnv

from fiery_b200 import _lib, install, ops  # noqa: F401
from fiery_b200.causal_conv import TensorCoreCausalConv3d, backward_weight_workspace_bytes
from fiery_b200.temporal import TensorCoreTemporalBlock
from oracle import temporal_oracle as TO
from tests._temporal_models import temporal_model


# ------------------------------------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------------------------------------
def _desc(b=3, s=3, X=200, Y=200, cin=35, cout=35, kt=2):
    d = _lib.CausalConv3dDesc()
    d.batch, d.frames, d.grid_x, d.grid_y, d.in_channels, d.out_channels, d.kt = b, s, X, Y, cin, cout, kt
    return d


def _calls(d, p=256):
    """every entry point, with dummy pointers (p) that a rejected call never touches"""
    lib = _lib.load()
    return {
        "pack": lambda: lib.fiery_causal_conv3d_pack_weights(d, p, p, None),
        "forward": lambda: lib.fiery_causal_conv3d_forward(d, p, p, p, None),
        "backward_data": lambda: lib.fiery_causal_conv3d_backward_data(d, p, p, p, None),
        "backward_weight": lambda: lib.fiery_causal_conv3d_backward_weight(d, p, p, p, p, None),
    }


@pytest.mark.parametrize("field,kw", [("in_channels", dict(cin=0)), ("in_channels", dict(cin=65)), ("out_channels", dict(cout=0)),
                                      ("out_channels", dict(cout=65)), ("kt", dict(kt=3)), ("kt", dict(kt=0)),
                                      ("grid_y", dict(Y=202)), ("grid_x", dict(X=0)), ("frames", dict(s=-1))],
                         ids=["cin0", "cin65", "cout0", "cout65", "kt3", "kt0", "Y%4", "X0", "s-1"])
def test_limits_are_rejected_naming_the_field(field, kw):
    d = _desc(**kw)
    lib = _lib.load()
    for name, call in _calls(d).items():
        assert call() == -1, name
        assert field in lib.fiery_last_error().decode(), name
    assert lib.fiery_causal_conv3d_packed_bytes(d) == 0
    assert lib.fiery_causal_conv3d_backward_weight_workspace_bytes(d) == 0


def test_null_pointers_are_rejected():
    lib = _lib.load()
    d = _desc()
    for name, call in _calls(d, p=None).items():
        assert call() == -1, name
        assert "NULL" in lib.fiery_last_error().decode(), name


def test_limits_themselves_are_accepted():
    lib = _lib.load()
    assert lib.fiery_causal_conv3d_packed_bytes(_desc(cin=64, cout=64, kt=2)) > 0
    assert lib.fiery_causal_conv3d_packed_bytes(_desc(cin=1, cout=1, kt=1, X=1, Y=4)) > 0


@pytest.mark.parametrize("batch,frames", [(0, 3), (3, 0), (0, 0)])
def test_zero_frames_is_a_successful_no_op(batch, frames):
    d = _desc(b=batch, s=frames)
    calls = _calls(d)
    assert calls["forward"]() == 0 and calls["backward_data"]() == 0
    assert _lib.load().fiery_causal_conv3d_backward_weight_workspace_bytes(d) == 0


def _packed_rule(cin, cout, kt):
    """forward pack (9 kt taps x ceil(round8(C_in) / 32) atoms x round8(C_out) rows x 32 floats) + the input gradient's, (in, out)
    swapped"""
    r8 = lambda c: -(-c // 8) * 8
    one = lambda n, k: 9 * kt * -(-r8(k) // 32) * r8(n) * 32 * 4
    return one(cout, cin) + one(cin, cout)


def _workspace_rule(b, s, X, Y, cin, cout, kt):
    """128 chunks at most of 32-pixel row runs; a chunk's partial is 9 kt x C_out x C_in floats"""
    tiles = b * s * X * -(-Y // 32)
    return min(tiles, 128) * 9 * kt * cout * cin * 4


@pytest.mark.parametrize("b,s,X,Y,cin,cout,kt", [(3, 3, 200, 200, 35, 35, 2), (3, 3, 200, 200, 35, 35, 1), (4, 3, 400, 200, 32, 32, 2),
                                                 (1, 1, 1, 4, 1, 8, 1), (1, 2, 3, 4, 64, 64, 2), (3, 5, 7, 12, 35, 64, 2)])
def test_workspace_and_pack_rules(b, s, X, Y, cin, cout, kt):
    assert backward_weight_workspace_bytes((b, cin, s, X, Y), cout, kt) == _workspace_rule(b, s, X, Y, cin, cout, kt)
    assert _lib.load().fiery_causal_conv3d_packed_bytes(_desc(b, s, X, Y, cin, cout, kt)) == _packed_rule(cin, cout, kt)


# ------------------------------------------------------------------------------------------------------------------------------
# module and install helper
# ------------------------------------------------------------------------------------------------------------------------------
class _Fiery(torch.nn.Module):
    def __init__(self, temporal_model):
        super().__init__()
        self.temporal_model = temporal_model


def _causal_modules(model):
    return [m for m in model.modules() if isinstance(m, (TO.CausalConv3d, TensorCoreCausalConv3d))]


@pytest.mark.parametrize("kt", [1, 2])
def test_adopted_module_keeps_keys_and_parameters(kt):
    ref = TO.CausalConv3d(35, 35, kernel_size=(kt, 3, 3))
    tc = TensorCoreCausalConv3d.from_module(ref)
    assert list(tc.state_dict()) == list(ref.state_dict())
    assert tc.conv.weight is ref.conv.weight and tc.norm is ref.norm and tc.pad is ref.pad and tc.activation is ref.activation
    with pytest.raises(ValueError, match="out_channels = 65"):
        TensorCoreCausalConv3d.from_module(TO.CausalConv3d(35, 65))
    with pytest.raises(ValueError, match="bias-free"):
        TensorCoreCausalConv3d.from_module(TO.CausalConv3d(8, 8, bias=True))


@pytest.mark.parametrize("inbetween", [0, 1])
@pytest.mark.parametrize("order", ["causal_only", "causal_first", "blocks_first"])
def test_install_finds_every_path(order, inbetween):
    model = _Fiery(temporal_model(70, 3, (8, 8), start_out_channels=64, inbetween_layers=inbetween))
    keys = list(model.state_dict())
    params = dict(model.named_parameters())
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        if order == "blocks_first":
            install.use_tensor_core_temporal_model(model)
        install.use_tensor_core_causal_convs(model)
        if order == "causal_first":
            install.use_tensor_core_temporal_model(model)
    convs = _causal_modules(model)
    assert len(convs) == 2 * 2 + 2 * inbetween
    assert all(isinstance(m, TensorCoreCausalConv3d) for m in convs)
    blocks = [b for b in model.temporal_model.model if "TemporalBlock" in type(b).__name__]
    assert all(isinstance(b, TensorCoreTemporalBlock) for b in blocks) == (order != "causal_only")
    assert list(model.state_dict()) == keys
    assert all(p is params[n] for n, p in model.named_parameters())       # adopted, not copied
    before = [id(m) for m in _causal_modules(model)]
    install.use_tensor_core_causal_convs(model)                            # idempotent
    assert [id(m) for m in _causal_modules(model)] == before and list(model.state_dict()) == keys


def test_install_warns_once_for_uncovered_modules():
    install._warned.clear()
    wide = temporal_model(130, 2, (8, 8), start_out_channels=64)          # half channels 65
    with pytest.warns(RuntimeWarning, match="in_channels = 65"):
        install.use_tensor_core_causal_convs(_Fiery(wide))
    assert not any(isinstance(m, TensorCoreCausalConv3d) for m in _causal_modules(wide))
    with warnings.catch_warnings():
        warnings.simplefilter("error")                                   # the same reasons do not warn twice
        install.use_tensor_core_causal_convs(_Fiery(wide))
    biased = temporal_model(16, 2, (8, 8), start_out_channels=8)
    biased.model[0].convolution_paths[1][1].conv = torch.nn.Conv3d(8, 8, (1, 3, 3), bias=True)
    with pytest.warns(RuntimeWarning, match="bias-free"):
        install.use_tensor_core_causal_convs(_Fiery(biased))
    assert isinstance(biased.model[0].convolution_paths[0][1], TensorCoreCausalConv3d)      # the covered one is swapped
    assert isinstance(biased.model[0].convolution_paths[1][1], TO.CausalConv3d)
    ident = _Fiery(torch.nn.Identity())
    assert install.use_tensor_core_causal_convs(ident) is ident


def test_uncovered_map_width_runs_the_reference_conv_on_cpu_shapes():
    """A map of Y % 4 != 0 takes the reference's pad and Conv3d, with one warning, and gives the reference module's result."""
    torch.manual_seed(0)
    ref = TO.CausalConv3d(8, 8).eval()
    tc = TensorCoreCausalConv3d.from_module(ref)
    x = torch.randn(2, 8, 3, 5, 5)
    with pytest.warns(RuntimeWarning, match="Y = 5"):
        got = tc(x)
    assert torch.equal(got, TO.CausalConv3d.forward(ref, x))


def test_swapped_module_follows_sync_batchnorm_conversion():
    model = _Fiery(temporal_model(70, 3, (8, 8), start_out_channels=64))
    install.use_tensor_core_causal_convs(model)
    conv = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    m = conv.temporal_model.model[0].convolution_paths[0][1]
    assert isinstance(m, TensorCoreCausalConv3d) and isinstance(m.norm, torch.nn.SyncBatchNorm)


# ------------------------------------------------------------------------------------------------------------------------------
# fakes
# ------------------------------------------------------------------------------------------------------------------------------
def test_fakes_trace_symbolically():
    """The forward's fake gives (b, C_out, s, X, Y) contiguous fp32, the backward's gives x's and the weight's shapes, or empty
    tensors for gradients not asked for; b and s stay symbolic."""
    def fwd_bwd(x, w, g):
        y = torch.ops.fiery_b200.causal_conv3d(x, w)
        gx, gw = torch.ops.fiery_b200.causal_conv3d_backward(g, x, w, True, True)
        gx0, gw1 = torch.ops.fiery_b200.causal_conv3d_backward(g, x, w, False, True)
        return y, gx, gw, gx0, gw1

    with FakeTensorMode(shape_env=ShapeEnv()):
        x = torch.empty(3, 35, 2, 8, 8, device="cuda")
        w = torch.empty(32, 35, 2, 3, 3, device="cuda")
        g = torch.empty(3, 32, 2, 8, 8, device="cuda")
        gm = make_fx(fwd_bwd, tracing_mode="symbolic")(x, w, g)
        y, gx, gw, gx0, gw1 = gm(x, w, g)
    assert tuple(y.shape) == (3, 32, 2, 8, 8) and y.is_contiguous() and y.dtype == torch.float32
    assert tuple(gx.shape) == tuple(x.shape) and tuple(gw.shape) == tuple(w.shape)
    assert gx0.numel() == 0 and tuple(gw1.shape) == tuple(w.shape)
    assert "fiery_b200.causal_conv3d" in str(gm.code) and "fiery_b200.causal_conv3d_backward" in str(gm.code)
