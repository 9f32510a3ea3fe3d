"""CPU: the fused BatchNorm3d swap (fiery_b200/batch_norm.py, install.use_fused_batch_norm) -- swap order and idempotence with the other
temporal swaps, state_dict keys and shared tensors, the modules it leaves alone, convert_sync_batchnorm after the swap, the running
statistics' update rules against nn.BatchNorm3d (in fp64, from the batch's mean and variance), the C ABI's argument checks and the
operators' fakes on fake tensors."""
import copy
import warnings

import pytest
import torch
import torch.nn as nn

from fiery_b200 import _lib, install, ops  # noqa: F401
from fiery_b200.batch_norm import FusedBatchNorm3d
from oracle import temporal_oracle as TO
from tests._temporal_models import temporal_model


def _holder(m):
    return type("M", (), {"temporal_model": m})()


def _norms(m):
    """(name, module) of every batch norm under the model, the pyramid pooling's apart"""
    return [(n, x) for n, x in m.named_modules() if isinstance(x, nn.modules.batchnorm._BatchNorm) and "pyramid_pooling" not in n]


ORDERS = [("bn", "entry", "causal", "pool"), ("entry", "causal", "pool", "bn"), ("causal", "bn", "pool"), ("bn",)]
SWAPS = {"bn": install.use_fused_batch_norm, "pool": install.use_tensor_core_pyramid_pooling,
         "entry": install.use_tensor_core_temporal_model, "causal": install.use_tensor_core_causal_convs}


@pytest.mark.parametrize("order", ORDERS, ids=lambda o: "-".join(o))
@pytest.mark.parametrize("inbetween", [0, 1])
def test_swap_order_idempotence_and_state_dict(order, inbetween):
    m = temporal_model(70, 3, (8, 8), start_out_channels=64, inbetween_layers=inbetween)
    keys = list(m.state_dict())
    tensors = {k: v for k, v in m.state_dict(keep_vars=True).items()}
    n_norms = len(_norms(m))
    h = _holder(m)
    for name in order:
        SWAPS[name](h)
    norms = _norms(m)
    assert len(norms) == n_norms and all(type(x) is FusedBatchNorm3d for _, x in norms)
    pp = [x for n, x in m.named_modules() if "pyramid_pooling" in n and isinstance(x, nn.modules.batchnorm._BatchNorm)]
    assert pp and all(type(x) is nn.BatchNorm3d for x in pp)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        install.use_fused_batch_norm(h)                               # a second call does nothing
    assert [x for _, x in _norms(m)] == [x for _, x in norms]
    assert list(m.state_dict()) == keys
    for k, v in m.state_dict(keep_vars=True).items():               # the same Parameter and buffer objects
        assert v is tensors[k], k


def test_sync_batch_norm_is_left_alone_with_one_warning():
    m = temporal_model(70, 3, (8, 8), start_out_channels=64)
    blk = m.model[0]
    sync = nn.SyncBatchNorm(blk.out_channels)
    blk.aggregation[0].norm = sync
    install._warned.clear()
    with pytest.warns(RuntimeWarning, match="SyncBatchNorm") as rec:
        install.use_fused_batch_norm(_holder(m))
    assert len(rec) == 1 and "aggregation.0.norm" in str(rec[0].message)
    assert blk.aggregation[0].norm is sync
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        install.use_fused_batch_norm(_holder(m))                      # the same skip warns once


def test_convert_sync_batchnorm_after_the_swap():
    m = temporal_model(70, 3, (8, 8), start_out_channels=64)
    install.use_tensor_core_temporal_model(_holder(m))
    install.use_fused_batch_norm(_holder(m))
    before = {k: v for k, v in m.state_dict(keep_vars=True).items()}
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(m)
    norms = _norms(conv)
    assert norms and all(type(x) is nn.SyncBatchNorm for _, x in norms)
    after = conv.state_dict(keep_vars=True)
    assert list(after) == list(before)
    for k, v in after.items():
        assert v is before[k] or torch.equal(v, before[k]), k
    for n, x in norms:
        assert x.weight is before[n + ".weight"] and x.running_mean is before[n + ".running_mean"]


@pytest.mark.parametrize("kw", [dict(), dict(momentum=None), dict(track_running_stats=False), dict(affine=False)],
                         ids=["momentum0.1", "cumulative", "untracked", "no-affine"])
def test_running_stat_update_matches_batch_norm(kw):
    torch.manual_seed(0)
    ref = nn.BatchNorm3d(5, **kw).double().train()
    mine = FusedBatchNorm3d(copy.deepcopy(ref))
    for step in range(3):
        x = torch.randn(2, 5, 3, 4, 6, dtype=torch.float64) * (step + 1) + step
        ref(x)
        mean = x.mean(dim=(0, 2, 3, 4))
        var = x.var(dim=(0, 2, 3, 4), unbiased=False)
        mine.update_running_stats(mean, var, x.numel() // 5)
    for (n, a), (_, b) in zip(mine.named_buffers(), ref.named_buffers()):
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-14), n
    assert [n for n, _ in mine.named_buffers()] == [n for n, _ in ref.named_buffers()]
    mine.eval()
    before = [b.clone() for b in mine.buffers()]
    mine.update_running_stats(mean, var, 10)                           # eval: nothing changes
    assert all(torch.equal(a, b) for a, b in zip(before, mine.buffers()))


def test_adopts_tensors_and_mode():
    bn = nn.BatchNorm3d(7, eps=1e-3, momentum=0.3).eval()
    f = FusedBatchNorm3d(bn)
    assert (f.weight is bn.weight and f.bias is bn.bias and f.running_mean is bn.running_mean and f.running_var is bn.running_var
            and f.num_batches_tracked is bn.num_batches_tracked)
    assert (f.eps, f.momentum, f.affine, f.track_running_stats, f.training) == (1e-3, 0.3, True, True, False)
    assert list(f.state_dict()) == list(bn.state_dict())
    f.load_state_dict(bn.state_dict())


# ------------------------------------------------------------------------------------------------------------------------------
# C ABI argument checks and fakes
# ------------------------------------------------------------------------------------------------------------------------------
def _desc(b=3, c=35, s=3, pixels=40000, training=1, relu=1, eps=1e-5, strides=None):
    d = _lib.BatchNormDesc()
    d.batch, d.channels, d.frames, d.pixels = b, c, s, pixels
    d.stride_b, d.stride_c, d.stride_t = strides or (c * s * pixels, s * pixels, pixels)
    d.training, d.relu, d.eps = training, relu, eps
    return d


BAD = [(dict(c=0), "channels"), (dict(b=0), "batch * frames"), (dict(s=-1), "batch"), (dict(pixels=0), "pixels"),
       (dict(strides=(-1, 0, 0)), "strides"), (dict(training=2), "training"), (dict(relu=-1), "relu"), (dict(eps=-1.0), "eps"),
       (dict(eps=float("nan")), "eps"), (dict(b=1, s=1, pixels=1), "must be >= 2 in training")]


@pytest.mark.parametrize("kw,needle", BAD, ids=[n for _, n in BAD])
def test_batch_norm_rejects(kw, needle):
    lib = _lib.load()
    d = _desc(**kw)
    assert lib.fiery_batch_norm_workspace_bytes(d) == 0
    assert lib.fiery_batch_norm_forward(d, 256, 0, 0, 0, 0, 0, 256, 256, 256, 256, None) != 0
    assert needle in lib.fiery_last_error().decode()
    assert lib.fiery_batch_norm_backward(d, 256, 256, 0, 0, 256, 256, 256, 0, 0, 256, None) != 0
    assert needle in lib.fiery_last_error().decode()


def test_batch_norm_rejects_pointers():
    lib = _lib.load()
    d = _desc()
    assert lib.fiery_batch_norm_forward(d, 0, 0, 0, 0, 0, 0, 256, 256, 256, 256, None) != 0
    assert "NULL" in lib.fiery_last_error().decode()
    assert lib.fiery_batch_norm_forward(d, 256, 0, 0, 0, 0, 0, 256, 256, 256, 260, None) != 0
    assert "16-byte" in lib.fiery_last_error().decode()
    d.training = 0
    assert lib.fiery_batch_norm_forward(d, 256, 0, 0, 0, 0, 0, 256, 256, 256, 256, None) != 0
    assert "running_mean" in lib.fiery_last_error().decode()
    assert lib.fiery_batch_norm_backward(d, 256, 0, 0, 0, 256, 256, 256, 0, 0, 256, None) != 0
    assert "NULL" in lib.fiery_last_error().decode()


def test_batch_norm_eval_takes_one_value_and_workspace_size():
    lib = _lib.load()
    assert lib.fiery_batch_norm_workspace_bytes(_desc(b=1, s=1, pixels=1, training=0)) > 0
    # 20-byte coefficients per channel in a 256-byte-rounded block, then 8 bytes per piece of 4096 pixels: 40000 -> 10 per plane
    assert lib.fiery_batch_norm_workspace_bytes(_desc()) == 768 + 35 * 9 * 10 * 8


def test_fakes_on_fake_tensors():
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        x = torch.empty(2, 3, 35, 8, 8, device="cuda", dtype=torch.float16).permute(0, 2, 1, 3, 4)
        w = torch.empty(35, device="cuda")
        y, mean, var = torch.ops.fiery_b200.batch_norm_act(x, w, w, None, None, None, True, 1e-5, True)
        assert y.shape == (2, 35, 3, 8, 8) and y.dtype == torch.float32 and y.is_contiguous()
        assert mean.shape == var.shape == (35,) and mean.dtype == torch.float32
        y, _, _ = torch.ops.fiery_b200.batch_norm_act(x, None, None, w, w, torch.empty(2, 35, 3, 8, 8, device="cuda"), False, 1e-5,
                                                     False)
        assert y.shape == (2, 35, 3, 8, 8) and y.is_contiguous()
        g = torch.empty(2, 35, 3, 8, 8, device="cuda")
        for need in ((True, True, True), (False, True, True), (True, False, False), (False, False, True)):
            dx, dw, db = torch.ops.fiery_b200.batch_norm_act_backward(g, x, w, w, w, w, True, 1e-5, True, *need)
            assert tuple(dx.shape) == ((2, 35, 3, 8, 8) if need[0] else (0,))
            assert dx.dtype == torch.float16 and (not need[0] or dx.is_contiguous())
            assert tuple(dw.shape) == ((35,) if need[1] else (0,)) and tuple(db.shape) == ((35,) if need[2] else (0,))
