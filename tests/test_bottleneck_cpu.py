"""The Bottleneck's host side without a GPU: which modules the kernels cover, the swap into a FuturePrediction, the operators'
fake shapes, and the C ABI's size functions and rejections."""
from __future__ import annotations

import copy

import pytest
import torch
import torch.nn as nn

from fiery_b200 import _lib, install
from fiery_b200 import bottleneck as bk
from fiery_b200.bottleneck import TensorCoreBottleneck, module_reason
from fiery_b200.future_prediction import TensorCoreSpatialGRU
from oracle.future_oracle import Bottleneck, FuturePrediction


class _Model(nn.Module):
    pass


def _model(c=64):
    torch.manual_seed(0)
    m = _Model()
    m.future_prediction = FuturePrediction(c, 32)
    return m


def _with(block, **layers):
    b = copy.deepcopy(block)
    for name, mod in layers.items():
        setattr(b.layers, name, mod)
    return b


def test_plain_bottleneck_is_covered():
    assert module_reason(Bottleneck(64)) is None
    assert module_reason(Bottleneck(2)) is None
    assert module_reason(Bottleneck(35)) is None


@pytest.mark.parametrize("variant", ["projection", "downsample", "upsample", "dropout", "kernel5", "sync", "c130", "relu6"])
def test_rejected_variants(variant):
    b = Bottleneck(64)
    if variant == "projection":
        b.projection = nn.Sequential(nn.Conv2d(64, 64, 1, bias=False), nn.BatchNorm2d(64))
    elif variant == "downsample":
        b = _with(b, conv=nn.Conv2d(32, 32, 3, stride=2, padding=1, bias=False))
    elif variant == "upsample":
        b = _with(b, conv=nn.ConvTranspose2d(32, 32, 3, stride=2, padding=1, output_padding=1, bias=False))
    elif variant == "dropout":
        b = _with(b, dropout=nn.Dropout2d(0.1))
    elif variant == "kernel5":
        b = Bottleneck(64, kernel_size=5)
    elif variant == "sync":
        b = nn.SyncBatchNorm.convert_sync_batchnorm(b)
    elif variant == "c130":
        b = Bottleneck(130)
    elif variant == "relu6":
        b = _with(b, abn=nn.Sequential(nn.BatchNorm2d(32), nn.ReLU6()))
    reason = module_reason(b)
    assert reason is not None
    with pytest.raises(ValueError):
        TensorCoreBottleneck.from_module(b)


def test_swap_takes_exactly_the_nine_bottlenecks_and_keeps_the_state_dict():
    m = _model()
    keys = list(m.state_dict().keys())
    params = {id(p) for p in m.parameters()}
    install.use_tensor_core_bottlenecks(m)
    fp = m.future_prediction
    assert sum(isinstance(x, TensorCoreBottleneck) for x in fp.modules()) == 9
    assert not any(isinstance(x, Bottleneck) for x in fp.modules())
    assert list(m.state_dict().keys()) == keys
    assert {id(p) for p in m.parameters()} == params
    swapped = [id(x) for x in fp.modules() if isinstance(x, TensorCoreBottleneck)]
    install.use_tensor_core_bottlenecks(m)
    assert [id(x) for x in fp.modules() if isinstance(x, TensorCoreBottleneck)] == swapped


@pytest.mark.parametrize("order", ["gru_first", "bottleneck_first"])
def test_swaps_work_in_either_order(order):
    m = _model()
    keys = list(m.state_dict().keys())
    swaps = [install.use_tensor_core_future_prediction, install.use_tensor_core_bottlenecks]
    for swap in (swaps if order == "gru_first" else swaps[::-1]):
        swap(m)
    fp = m.future_prediction
    assert sum(isinstance(x, TensorCoreSpatialGRU) for x in fp.modules()) == 3
    assert sum(isinstance(x, TensorCoreBottleneck) for x in fp.modules()) == 9
    assert list(m.state_dict().keys()) == keys


def test_model_without_future_prediction_is_untouched():
    m = _Model()
    assert install.use_tensor_core_bottlenecks(m) is m


def test_uncovered_bottleneck_is_left_with_one_warning():
    m = _model()
    m.future_prediction.res_blocks[1][2].layers.dropout = nn.Dropout2d(0.2)
    _lib._warned.clear()
    with pytest.warns(RuntimeWarning, match=r"res_blocks\[1\]\[2\]"):
        install.use_tensor_core_bottlenecks(m)
    assert isinstance(m.future_prediction.res_blocks[1][2], Bottleneck)
    assert sum(isinstance(x, TensorCoreBottleneck) for x in m.future_prediction.modules()) == 8


def test_cpu_input_runs_the_reference_with_a_warning():
    torch.manual_seed(0)
    ref = Bottleneck(16)
    ours = TensorCoreBottleneck.from_module(copy.deepcopy(ref))
    x = torch.randn(2, 16, 8, 8)
    _lib._warned.clear()
    with pytest.warns(RuntimeWarning, match="CPU input"):
        out = ours(x)
    torch.testing.assert_close(out, copy.deepcopy(ref)(x))


def test_fake_shapes():
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        x = torch.empty(12, 35, 20, 24, device="cuda")
        wd, wc, wu = torch.empty(17, 35, 1, 1, device="cuda"), torch.empty(17, 17, 3, 3, device="cuda"), torch.empty(35, 17, 1, 1,
                                                                                                                     device="cuda")
        norms = [torch.empty(k, device="cuda") for k in (17,) * 4 + (17,) * 4 + (35,) * 4]
        out, y1, y2, y3, stats = torch.ops.fiery_b200.bottleneck(x, wd, wc, wu, *norms, True, 1e-5)
        assert out.shape == (12, 35, 20, 24) and y1.shape == y2.shape == (12, 17, 20, 24) and y3.shape == out.shape
        assert stats.shape == (2 * (17 + 17 + 35),) and out.dtype == torch.float32
        need = [True, False, True, True, False, True, True, True, False, True]
        g = torch.ops.fiery_b200.bottleneck_backward(out, x, y1, y2, y3, stats, wd, wc, wu, norms[0], norms[1], norms[4], norms[5],
                                                     norms[8], norms[9], True, 1e-5, need)
        likes = [x, wd, wc, wu, norms[0], norms[1], norms[4], norms[5], norms[8], norms[9]]
        for gi, like, nd in zip(g, likes, need):
            assert gi.shape == (like.shape if nd else (0,))


def test_size_functions():
    lib = _lib.load()
    maps, h, w, c = 12, 200, 200, 64
    packed, fwd, bwd = bk.workspace_bytes(maps, h, w, c)
    assert packed > 0 and fwd > 0
    m, p = c // 2, h * w
    assert bwd >= 4 * maps * p * (c + 2 * m)               # dy3 and the two (maps, M) gradient buffers
    assert bk.workspace_bytes(12, 200, 200, 128)[0] > packed
    assert lib.fiery_bottleneck_packed_bytes(bk.desc(1, 4, 4, 64)) == bk.workspace_bytes(1, 4, 4, 64)[0] == packed


@pytest.mark.parametrize("field,value,message", [
    ("channels", 1, "channels = 1 must be in 2..128"),
    ("channels", 130, "channels = 130 must be in 2..128"),
    ("grid_y", 10, "grid_y = 10 must be a positive multiple of 4"),
    ("grid_x", 0, "grid_x = 0 must be >= 1"),
    ("maps", 0, "maps = 0 must be >= 1"),
    ("training", 2, "training = 2 must be 0 or 1"),
    ("eps", -1.0, "eps = -1 must be >= 0"),
])
def test_rejected_descriptors(field, value, message):
    lib = _lib.load()
    d = bk.desc(2, 8, 8, 64)
    setattr(d, field, value)
    assert lib.fiery_bottleneck_packed_bytes(d) == 0
    assert lib.fiery_bottleneck_forward_workspace_bytes(d) == 0
    assert lib.fiery_bottleneck_backward_workspace_bytes(d) == 0
    assert lib.fiery_bottleneck_forward(d, *([None] * 10)) != 0
    assert message in lib.fiery_last_error().decode()


def test_null_pointers_are_rejected():
    lib = _lib.load()
    assert lib.fiery_bottleneck_forward(bk.desc(1, 1, 4, 64), *([None] * 10)) != 0
    assert "NULL pointer" in lib.fiery_last_error().decode()
    d = bk.desc(1, 1, 4, 64)
    d.grid_x, d.grid_y = 1, 4
    d.maps = 1
    assert lib.fiery_bottleneck_backward(d, *([None] * 16)) != 0
    assert "NULL pointer" in lib.fiery_last_error().decode()
