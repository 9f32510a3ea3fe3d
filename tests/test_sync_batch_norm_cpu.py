"""CPU: the swap to FusedSyncBatchNorm (install.use_fused_sync_batch_norm), the GRU's coverage of it, the argument checks of the
group entries (fiery_batch_norm_*_gathered, fiery_spatial_gru_*_step_*), and a numpy model of the rank-order merge."""
from __future__ import annotations

import ctypes
import warnings

import numpy as np
import pytest
import torch
import torch.nn as nn

from fiery_b200 import _lib, install
from fiery_b200.batch_norm import FusedBatchNorm3d, FusedSyncBatchNorm
from fiery_b200.future_prediction import TensorCoreSpatialGRU, module_reason
from oracle.future_oracle import FuturePrediction
from oracle.temporal_oracle import TemporalModel


class _Holder(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.temporal_model = TemporalModel(8, 3, (6, 8), start_out_channels=8)
        self.future_prediction = FuturePrediction(8, 4, n_gru_blocks=3, n_res_layers=1)


def _converted():
    return nn.SyncBatchNorm.convert_sync_batchnorm(_Holder())


def _fused(m):
    return [(n, x) for n, x in m.named_modules() if isinstance(x, FusedSyncBatchNorm)]


def test_swap_replaces_the_temporal_norms_and_the_gru_norms_only():
    m = _converted()
    keys = {k: v for k, v in m.state_dict(keep_vars=True).items()}
    install.use_fused_sync_batch_norm(m)
    fused = dict(_fused(m))
    assert fused and all(type(x) is FusedSyncBatchNorm for x in fused.values())
    assert not any("pyramid_pooling" in n for n in fused)
    assert all(type(x) is nn.SyncBatchNorm for n, x in m.named_modules() if "pyramid_pooling" in n and isinstance(x, nn.SyncBatchNorm))
    assert sum(n.startswith("future_prediction.spatial_grus") for n in fused) == 3
    assert not any(n.startswith("future_prediction.res_blocks") for n in fused)         # the Bottlenecks stay torch's
    after = m.state_dict(keep_vars=True)
    assert list(after) == list(keys) and all(after[k] is keys[k] for k in keys)       # same tensors, same keys
    assert all(isinstance(x, nn.SyncBatchNorm) for x in fused.values())


def test_process_group_is_adopted():
    bn = nn.SyncBatchNorm(4, process_group="group-object")
    f = FusedSyncBatchNorm(bn)
    assert f.process_group == "group-object" and f.weight is bn.weight and f.running_var is bn.running_var
    assert f.num_batches_tracked is bn.num_batches_tracked


@pytest.mark.parametrize("order", ["sync_first", "sync_last", "between"])
def test_idempotent_in_every_order_with_the_other_swaps(order):
    m = _converted()
    others = [install.use_tensor_core_temporal_model, install.use_tensor_core_causal_convs, install.use_tensor_core_pyramid_pooling,
              install.use_fused_batch_norm, install.use_tensor_core_future_prediction]
    seq = {"sync_first": [install.use_fused_sync_batch_norm] + others, "sync_last": others + [install.use_fused_sync_batch_norm],
           "between": others[:2] + [install.use_fused_sync_batch_norm] + others[2:]}[order]
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        for fn in seq + seq:
            fn(m)
    ids = [(n, id(x)) for n, x in _fused(m)]
    install.use_fused_sync_batch_norm(m)
    assert [(n, id(x)) for n, x in _fused(m)] == ids
    grus = list(m.future_prediction.spatial_grus)
    if order != "sync_last":
        assert all(isinstance(g, TensorCoreSpatialGRU) for g in grus)
    assert all(isinstance(g.conv_state_tilde.norm, FusedSyncBatchNorm) for g in grus)
    assert not any("SyncBatchNorm module(s) left" in str(w.message) for w in rec if order == "sync_first")


def test_use_fused_batch_norm_neither_touches_nor_warns_about_a_fused_sync_norm():
    m = _converted()
    install.use_fused_sync_batch_norm(m)
    before = [(n, id(x)) for n, x in _fused(m)]
    _lib._warned.clear()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        install.use_fused_batch_norm(m)
    assert [(n, id(x)) for n, x in _fused(m)] == before
    assert not any("SyncBatchNorm" in str(w.message) for w in rec)
    assert not any(isinstance(x, FusedBatchNorm3d) for x in m.modules())


def test_gru_swap_after_the_sync_swap_and_module_reason():
    m = _converted()
    gru = m.future_prediction.spatial_grus[0]
    assert "SyncBatchNorm" in module_reason(gru)
    install.use_fused_sync_batch_norm(m)
    assert module_reason(gru) is None
    install.use_tensor_core_future_prediction(m)
    assert all(isinstance(g, TensorCoreSpatialGRU) for g in m.future_prediction.spatial_grus)


# ------------------------------------------------------------------------------------------------------------------------------
# the C entries reject bad arguments before touching the device
# ------------------------------------------------------------------------------------------------------------------------------
def _bn_desc(**kw):
    d = _lib.BatchNormDesc()
    d.batch, d.channels, d.frames, d.pixels = 2, 4, 1, 16
    d.stride_b, d.stride_c, d.stride_t = 64, 16, 16
    d.training, d.relu, d.eps = 1, 1, 1e-5
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _err(rc, *words):
    assert rc != 0
    msg = _lib.load().fiery_last_error().decode()
    for w in words:
        assert w in msg, msg


P, P8 = 1 << 20, (1 << 20) + 8                                  # fake 16-byte and 8-byte aligned addresses, never dereferenced


def test_batch_norm_group_entries_reject_bad_arguments():
    lib = _lib.load()
    _err(lib.fiery_batch_norm_local_stats(_bn_desc(training=0), P, P, P, None), "training")
    _err(lib.fiery_batch_norm_local_stats(_bn_desc(batch=-1), P, P, P, None), "batch")
    _err(lib.fiery_batch_norm_local_stats(_bn_desc(), P, P + 4, P, None), "aligned")
    _err(lib.fiery_batch_norm_local_stats(_bn_desc(), P, None, P, None), "NULL")
    _err(lib.fiery_batch_norm_forward_gathered(_bn_desc(), 0, P, P, 0, 0, 0, P, P, P, 0, P, None), "world")
    _err(lib.fiery_batch_norm_forward_gathered(_bn_desc(), 2, None, P, 0, 0, 0, P, P, P, 0, P, None), "gathered")
    _err(lib.fiery_batch_norm_forward_gathered(_bn_desc(), 2, P + 4, P, 0, 0, 0, P, P, P, 0, P, None), "gathered", "aligned")
    _err(lib.fiery_batch_norm_forward_gathered(_bn_desc(), 2, P, P, 0, 0, 0, None, P, P, 0, P, None), "NULL")
    _err(lib.fiery_batch_norm_local_grad_sums(_bn_desc(relu=2), P, P, 0, 0, P, P, P, 0, 0, P, None), "relu")
    _err(lib.fiery_batch_norm_local_grad_sums(_bn_desc(), P, P, 0, 0, P, P, None, 0, 0, P, None), "NULL")
    _err(lib.fiery_batch_norm_backward_gathered(_bn_desc(), -1, P, P, P, 0, 0, P, P, P, P, None), "world")
    _err(lib.fiery_batch_norm_backward_gathered(_bn_desc(eps=-1.0), 1, P, P, P, 0, 0, P, P, P, P, None), "eps")
    assert lib.fiery_batch_norm_sync_workspace_bytes(_bn_desc(training=0)) == 0
    # an empty rank is a valid member of a group, but not of a single-rank call
    assert lib.fiery_batch_norm_sync_workspace_bytes(_bn_desc(batch=0)) > 0
    assert lib.fiery_batch_norm_workspace_bytes(_bn_desc(batch=0)) == 0


def _gru_desc(**kw):
    from fiery_b200.future_prediction import _desc
    d = _desc(2, 3, 3, 8, 8, 4, 4)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_spatial_gru_step_entries_reject_bad_arguments():
    lib = _lib.load()
    _err(lib.fiery_spatial_gru_forward_step_begin(_gru_desc(training=0), 0, P, P, P, P, P, P, P8, P, None), "training")
    _err(lib.fiery_spatial_gru_forward_step_begin(_gru_desc(), 3, P, P, P, P, P, P, P8, P, None), "t = 3")
    _err(lib.fiery_spatial_gru_forward_step_begin(_gru_desc(), -1, P, P, P, P, P, P, P8, P, None), "t = -1")
    _err(lib.fiery_spatial_gru_forward_step_begin(_gru_desc(), 0, P + 4, P, P, P, P, P, P8, P, None), "16-byte")
    _err(lib.fiery_spatial_gru_forward_step_begin(_gru_desc(), 0, P, P, P, P, P, P, P + 4, P, None), "stats")
    _err(lib.fiery_spatial_gru_forward_step_end(_gru_desc(), 0, 0, P8, P, 0, 0, P, P, P, P, 0, P, None), "world")
    _err(lib.fiery_spatial_gru_forward_step_end(_gru_desc(), 0, 2, None, P, 0, 0, P, P, P, P, 0, P, None), "gathered")
    _err(lib.fiery_spatial_gru_forward_step_end(_gru_desc(h_channels=65), 0, 2, P8, P, 0, 0, P, P, P, P, 0, P, None), "h_channels")
    _err(lib.fiery_spatial_gru_backward_step_begin(_gru_desc(), 0, P, P, P, P, P, P, P, 0, 0, P + 4, P8, P, None), "16-byte")
    _err(lib.fiery_spatial_gru_backward_step_begin(_gru_desc(), 0, P, P, P, P, P, P, P, 0, 0, 0, None, P, None), "NULL")
    _err(lib.fiery_spatial_gru_backward_step_end(_gru_desc(), 0, 0, P8, P, P, P, P, P, P, 0, 0, 0, 0, P, None), "world")
    _err(lib.fiery_spatial_gru_backward_step_end(_gru_desc(grid_y=6), 0, 1, P8, P, P, P, P, P, P, 0, 0, 0, 0, P, None), "grid_y")
    _err(lib.fiery_spatial_gru_backward_weights(_gru_desc(training=0), P, P, P, P, P, 0, 0, 0, 0, 0, P, None), "training")
    _err(lib.fiery_spatial_gru_backward_weights(_gru_desc(), None, P, P, P, P, 0, 0, 0, 0, 0, P, None), "NULL")


# ------------------------------------------------------------------------------------------------------------------------------
# the rank-order merge, restated in numpy, against fp64 brute force
# ------------------------------------------------------------------------------------------------------------------------------
def merge_forward(triplets):
    """(world, C, 3) (n, mean, M2) -> (n, mean, M2) per channel: rank 0's triplet, then Chan's formula rank by rank, n = 0 skipped"""
    n, m, m2 = triplets[0, :, 0].copy(), triplets[0, :, 1].copy(), triplets[0, :, 2].copy()
    for t in triplets[1:]:
        nb = t[:, 0]
        ok = nb != 0
        nn_ = np.where(ok, n + nb, 1.0)
        delta = t[:, 1] - m
        m = np.where(ok, m + delta * (nb / nn_), m)
        m2 = np.where(ok, m2 + t[:, 2] + delta * delta * (n * nb / nn_), m2)
        n = np.where(ok, n + nb, n)
    return n, m, m2


@pytest.mark.parametrize("sizes", [[7], [3, 0, 5], [0, 4, 1, 9], [1, 1], [0, 6]])
def test_rank_order_merge_matches_brute_force(sizes):
    rng = np.random.default_rng(sum(sizes))
    c = 5
    shards = [rng.normal(3.0, 2.0, size=(s, c)) for s in sizes]
    trip = np.stack([np.stack([np.full(c, float(len(s))), s.mean(0) if len(s) else np.zeros(c),
                               ((s - s.mean(0)) ** 2).sum(0) if len(s) else np.zeros(c)], axis=1) for s in shards])
    n, m, m2 = merge_forward(trip)
    whole = np.concatenate(shards)
    assert np.all(n == len(whole))
    np.testing.assert_allclose(m, whole.mean(0), rtol=1e-13)
    np.testing.assert_allclose(m2 / n, whole.var(0), rtol=1e-12)
    # the backward's sums: plain sums over the ranks
    s1 = sum(s.sum(0) for s in shards)
    np.testing.assert_allclose(s1, whole.sum(0), rtol=1e-13)
    # a single rank: its own triplet, untouched
    one = merge_forward(trip[:1])
    assert all(np.array_equal(a, b) for a, b in zip(one, (trip[0, :, 0], trip[0, :, 1], trip[0, :, 2])))


def test_swap_of_a_model_with_future_prediction_only():
    holder = nn.Module()
    holder.future_prediction = nn.SyncBatchNorm.convert_sync_batchnorm(FuturePrediction(8, 4, n_gru_blocks=2, n_res_layers=1))
    install.use_fused_sync_batch_norm(holder)
    install.use_tensor_core_future_prediction(holder)
    assert all(isinstance(g, TensorCoreSpatialGRU) and isinstance(g.conv_state_tilde.norm, FusedSyncBatchNorm)
               for g in holder.future_prediction.spatial_grus)
