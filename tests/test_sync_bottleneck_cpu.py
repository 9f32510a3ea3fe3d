"""CPU: the swap of converted Bottlenecks onto the kernels (install.use_tensor_core_sync_bottlenecks), which blocks and norm kinds
module_reason accepts, and the argument checks of the group stages (fiery_bottleneck_sync_*_stage)."""
from __future__ import annotations

import copy
import itertools
import warnings

import pytest
import torch
import torch.nn as nn

from fiery_b200 import _lib, install
from fiery_b200 import bottleneck as bk
from fiery_b200.batch_norm import FusedSyncBatchNorm
from fiery_b200.bottleneck import TensorCoreBottleneck, module_reason
from fiery_b200.future_prediction import TensorCoreSpatialGRU
from oracle.future_oracle import Bottleneck, FuturePrediction
from oracle.temporal_oracle import TemporalModel


class _Holder(nn.Module):
    def __init__(self, temporal: bool):
        super().__init__()
        torch.manual_seed(0)
        if temporal:
            self.temporal_model = TemporalModel(8, 3, (6, 8), start_out_channels=8)
        self.future_prediction = FuturePrediction(16, 4)


def _converted(temporal=False, group="group-object"):
    return nn.SyncBatchNorm.convert_sync_batchnorm(_Holder(temporal), process_group=group)


def _res_norms(m):
    return [(n, x) for n, x in m.future_prediction.res_blocks.named_modules() if isinstance(x, nn.SyncBatchNorm)]


@pytest.mark.parametrize("temporal", [False, True], ids=["alone", "with_temporal"])
def test_swap_takes_the_nine_blocks_and_their_27_norms(temporal):
    m = _converted(temporal)
    keys = m.state_dict(keep_vars=True)
    install.use_tensor_core_sync_bottlenecks(m)
    fp = m.future_prediction
    assert sum(isinstance(x, TensorCoreBottleneck) for x in fp.modules()) == 9
    assert not any(isinstance(x, Bottleneck) for x in fp.modules())
    norms = _res_norms(m)
    assert len(norms) == 27 and all(type(x) is FusedSyncBatchNorm for _, x in norms)
    assert all(x.process_group == "group-object" for _, x in norms)
    after = m.state_dict(keep_vars=True)
    assert list(after) == list(keys) and all(after[k] is keys[k] for k in keys)       # same tensors, same keys
    # nothing outside the Bottlenecks is touched
    assert all(type(x) is nn.SyncBatchNorm for n, x in m.named_modules() if isinstance(x, nn.SyncBatchNorm)
               and not n.startswith("future_prediction.res_blocks"))
    assert all(module_reason(x) is None for x in fp.modules() if isinstance(x, TensorCoreBottleneck))


SWAPS = ["use_tensor_core_sync_bottlenecks", "use_fused_sync_batch_norm", "use_tensor_core_future_prediction",
         "use_tensor_core_bottlenecks"]


@pytest.mark.parametrize("order", list(itertools.permutations(range(4))), ids=lambda o: "-".join(map(str, o)))
def test_idempotent_in_every_order_with_the_other_swaps(order):
    m = _converted(temporal=True)
    keys = list(m.state_dict())
    seq = [getattr(install, SWAPS[i]) for i in order]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for fn in seq:
            fn(m)
        blocks = [(n, id(x)) for n, x in m.named_modules() if isinstance(x, (TensorCoreBottleneck, FusedSyncBatchNorm))]
        for fn in seq:
            fn(m)
    assert [(n, id(x)) for n, x in m.named_modules() if isinstance(x, (TensorCoreBottleneck, FusedSyncBatchNorm))] == blocks
    fp = m.future_prediction
    assert sum(isinstance(x, TensorCoreBottleneck) for x in fp.modules()) == 9
    assert len(_res_norms(m)) == 27 and all(type(x) is FusedSyncBatchNorm for _, x in _res_norms(m))
    assert all(isinstance(g, TensorCoreSpatialGRU) for g in fp.spatial_grus)
    assert not any(type(x) is nn.SyncBatchNorm for x in fp.modules())
    assert list(m.state_dict()) == keys


@pytest.mark.parametrize("variant", ["dropout", "projection"])
def test_an_uncovered_block_is_left_with_one_warning_naming_its_slot(variant):
    m = _Holder(temporal=False)
    block = m.future_prediction.res_blocks[1][2]
    if variant == "dropout":
        block.layers.dropout = nn.Dropout2d(0.2)
    else:
        block.projection = nn.Sequential(nn.Conv2d(16, 16, 1, bias=False), nn.BatchNorm2d(16))
    m = nn.SyncBatchNorm.convert_sync_batchnorm(m)
    _lib._warned.clear()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        install.use_tensor_core_sync_bottlenecks(m)
        install.use_tensor_core_sync_bottlenecks(m)
    hits = [w for w in rec if "res_blocks[1][2]" in str(w.message)]
    assert len(hits) == 1 and len(rec) == 1
    left = m.future_prediction.res_blocks[1][2]
    assert type(left) is Bottleneck
    assert all(type(x) is nn.SyncBatchNorm for x in left.layers.modules() if isinstance(x, nn.SyncBatchNorm))
    assert sum(isinstance(x, TensorCoreBottleneck) for x in m.future_prediction.modules()) == 8


def test_blocks_without_a_sync_norm_and_models_without_future_prediction_are_untouched():
    m = _Holder(temporal=False)
    before = [(n, id(x)) for n, x in m.named_modules()]
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        install.use_tensor_core_sync_bottlenecks(m)
    assert [(n, id(x)) for n, x in m.named_modules()] == before
    bare = nn.Module()
    assert install.use_tensor_core_sync_bottlenecks(bare) is bare


def test_use_fused_sync_batch_norm_still_leaves_the_bottleneck_norms_alone():
    m = _converted(temporal=True)
    install.use_fused_sync_batch_norm(m)
    assert len(_res_norms(m)) == 27 and all(type(x) is nn.SyncBatchNorm for _, x in _res_norms(m))


def test_a_swapped_tensor_core_block_converted_afterwards_takes_the_swap():
    m = _Holder(temporal=False)
    install.use_tensor_core_bottlenecks(m)
    ids = [id(x) for x in m.future_prediction.modules() if isinstance(x, TensorCoreBottleneck)]
    m = nn.SyncBatchNorm.convert_sync_batchnorm(m)
    install.use_tensor_core_sync_bottlenecks(m)
    assert [id(x) for x in m.future_prediction.modules() if isinstance(x, TensorCoreBottleneck)] == ids
    assert len(_res_norms(m)) == 27 and all(type(x) is FusedSyncBatchNorm for _, x in _res_norms(m))


def test_module_reason_takes_one_norm_kind():
    plain = Bottleneck(16)
    assert module_reason(plain) is None
    converted = nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    assert "SyncBatchNorm" in module_reason(converted)
    fused = copy.deepcopy(converted)
    for abn in (fused.layers.abn_down_project, fused.layers.abn, fused.layers.abn_up_project):
        abn[0] = FusedSyncBatchNorm(abn[0])
    assert module_reason(fused) is None
    assert TensorCoreBottleneck.from_module(fused).layers is fused.layers
    mixed = copy.deepcopy(plain)
    mixed.layers.abn[0] = FusedSyncBatchNorm(nn.SyncBatchNorm(8))
    assert "different kinds" in module_reason(mixed)
    half = copy.deepcopy(fused)
    half.layers.abn_up_project[0] = nn.SyncBatchNorm(16)
    assert "SyncBatchNorm" in module_reason(half)
    with pytest.raises(ValueError):
        TensorCoreBottleneck.from_module(mixed)


def test_backward_gathers_depend_on_the_flags_only():
    params = [torch.ones(1)] * 6
    assert bk.sync_stages([True] + [False] * 9, params) == 3
    assert bk.sync_stages([False, True] + [False] * 8, params) == 3
    assert bk.sync_stages([False, False, True] + [False] * 7, params) == 2
    assert bk.sync_stages([False] * 3 + [True] + [False] * 6, params) == 1
    for k, stage in zip(range(4, 10), (2, 2, 1, 1, 0, 0)):
        assert bk.sync_stages([j == k for j in range(10)], params) == stage
    assert bk.sync_stages([False] * 4 + [True] * 2 + [False] * 4, [None] * 6) == 0   # a norm without affine parameters asks nothing


# ------------------------------------------------------------------------------------------------------------------------------
# the C entries reject bad arguments before touching the device
# ------------------------------------------------------------------------------------------------------------------------------
P, P8 = 1 << 20, (1 << 20) + 8                                  # fake 16-byte and 8-byte aligned addresses, never dereferenced


def _err(rc, *words):
    assert rc != 0
    msg = _lib.load().fiery_last_error().decode()
    for w in words:
        assert w in msg, msg


def _desc(**kw):
    d = bk.desc(2, 8, 8, 16)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _fwd(d, stage=1, world=2, gathered=P8, x=P, counts=P8, local=P8):
    """fiery_bottleneck_sync_forward_stage with every other pointer valid"""
    return _lib.load().fiery_bottleneck_sync_forward_stage(d, stage, world, gathered, x, P, bk._pointers([None] * 12), P, P, P, P, P,
                                                           counts, local, P, None)


def _bwd(d, stage=1, world=2, gathered=P8, grad_out=P, local=P8):
    return _lib.load().fiery_bottleneck_sync_backward_stage(d, stage, world, gathered, grad_out, P, P, P, P, P, P, bk._pointers([None] * 12),
                                                            P, 0, 0, 0, bk._pointers([None] * 6), local, P, None)


def test_group_stages_reject_bad_arguments():
    for call in (_fwd, _bwd):
        _err(call(_desc(training=0)), "training = 0 must be 1")
        _err(call(_desc(channels=130)), "channels = 130")
        _err(call(_desc(grid_y=6)), "grid_y = 6")
        _err(call(_desc(), stage=4), "stage = 4 must be in 0..3")
        _err(call(_desc(), stage=-1), "stage = -1")
        _err(call(_desc(), world=0), "world = 0 must be >= 1")
        _err(call(_desc(), gathered=None), "NULL gathered")
        _err(call(_desc(), gathered=P + 4), "gathered must be 8-byte aligned")
        _err(call(_desc(), local=None), "NULL local")
        _err(call(_desc(), local=P + 4), "local must be 8-byte aligned")
        _err(call(_desc(), stage=0, local=None), "NULL local")
    _err(_fwd(_desc(), x=None), "NULL pointer")
    _err(_fwd(_desc(), x=P + 4), "16-byte aligned")
    _err(_fwd(_desc(), counts=None), "NULL counts")
    _err(_fwd(_desc(), stage=3, counts=P + 4), "counts must be 8-byte aligned")
    _err(_bwd(_desc(), grad_out=None), "NULL pointer")
    _err(_bwd(_desc(), grad_out=P + 4), "16-byte aligned")
