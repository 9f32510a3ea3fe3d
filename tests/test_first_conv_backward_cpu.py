"""Host-side parts of the first BEV convolution's backward that need no GPU: the module swap of
``install.use_tensor_core_first_conv`` and the weight-gradient workspace rule of the C ABI."""
import warnings

import pytest
import torch
import torch.nn as nn

from fiery_b200 import _lib
from fiery_b200.bev_conv import FirstConv
from fiery_b200.install import use_tensor_core_first_conv


class _Decoder(nn.Module):
    def __init__(self, in_channels=64):
        super().__init__()
        self.first_conv = nn.Conv2d(in_channels, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)


class _Model(nn.Module):
    def __init__(self, in_channels=64):
        super().__init__()
        self.decoder = _Decoder(in_channels)


def test_swap_shares_the_parameter_and_keeps_state_dict_keys():
    m = _Model()
    weight = m.decoder.first_conv.weight
    keys = list(m.state_dict().keys())
    bn1, relu = m.decoder.bn1, m.decoder.relu
    assert use_tensor_core_first_conv(m) is m
    fc = m.decoder.first_conv
    assert isinstance(fc, FirstConv) and fc.bn is None and fc.relu is False
    assert fc.weight is weight
    assert list(m.state_dict().keys()) == keys
    assert m.decoder.bn1 is bn1 and m.decoder.relu is relu
    assert sum(p is weight for p in m.parameters()) == 1
    use_tensor_core_first_conv(m)                                   # idempotent
    assert m.decoder.first_conv is fc and fc.weight is weight


def test_swap_leaves_an_uncovered_layer_with_one_warning():
    m = _Model(in_channels=70)
    conv = m.decoder.first_conv
    with pytest.warns(RuntimeWarning, match="first_conv"):
        use_tensor_core_first_conv(m)
    assert m.decoder.first_conv is conv
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        use_tensor_core_first_conv(m)                               # warned once
    assert m.decoder.first_conv is conv


def _workspace_rule(n, h, w):
    """Python mirror of fiery_bev_first_conv_backward_weight_workspace_bytes: one (49, 64, 64) fp32 partial per pixel chunk,
    min(16 x 8 output tiles, 18) chunks."""
    if n < 0 or h < 1 or w < 1:
        return 0
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    tiles = n * ((wo + 15) // 16) * ((ho + 7) // 8)
    return min(tiles, 18) * 49 * 64 * 64 * 4


@pytest.mark.parametrize("n,h,w", [(0, 200, 200), (1, 1, 1), (1, 16, 32), (2, 33, 65), (3, 101, 99), (1, 250, 200), (8, 200, 200),
                                   (12, 400, 200), (1, 32, 64), (2, 31, 31)])
def test_workspace_bytes_follow_the_rule(n, h, w):
    lib = _lib.load()
    got = lib.fiery_bev_first_conv_backward_weight_workspace_bytes(n, h, w)
    assert got == _workspace_rule(n, h, w)
    assert got <= 18 * 49 * 64 * 64 * 4


@pytest.mark.parametrize("n,h,w", [(-1, 8, 8), (1, 0, 8), (1, 8, 0), (1, -5, 8)])
def test_workspace_bytes_reject_bad_shapes(n, h, w):
    assert _lib.load().fiery_bev_first_conv_backward_weight_workspace_bytes(n, h, w) == 0


def test_backward_entry_points_reject_bad_arguments_before_touching_a_device():
    lib = _lib.load()
    assert lib.fiery_bev_first_conv_backward_data(-1, 8, 8, 16, 16, 16, None) == -1         # FIERY_E_INVALID
    assert b"bad shape" in lib.fiery_last_error()
    assert lib.fiery_bev_first_conv_backward_data(1, 8, 8, None, 16, 16, None) == -1
    assert b"NULL" in lib.fiery_last_error()
    assert lib.fiery_bev_first_conv_backward_data(1, 8, 8, 16, 16, 20, None) == -1
    assert b"aligned" in lib.fiery_last_error()
    assert lib.fiery_bev_first_conv_backward_weight(1, 0, 8, 16, 16, 16, 16, None) == -1
    assert b"bad shape" in lib.fiery_last_error()
    assert lib.fiery_bev_first_conv_backward_weight(1, 8, 8, 16, 16, None, 16, None) == -1
    assert b"NULL" in lib.fiery_last_error()
    assert lib.fiery_bev_first_conv_backward_weight(1, 8, 8, 16, 16, 16, None, None) == -1
    assert b"NULL" in lib.fiery_last_error()
    assert lib.fiery_bev_first_conv_backward_weight(1, 8, 8, 16, 24, 16, 16, None) == -1
    assert b"aligned" in lib.fiery_last_error()
    assert lib.fiery_bev_conv_pack_weights_transposed(None, 16, None) == -1
