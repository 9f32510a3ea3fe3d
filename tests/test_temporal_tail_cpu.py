"""CPU: the temporal block's pyramid pooling and aggregation swap (fiery_b200/temporal.py, install.use_tensor_core_pyramid_pooling) --
coverage reasons, swap order and idempotence, state_dict keys, warnings, the pooled vector's arithmetic against the reference pooling
(from torch means, in fp64), the C ABI's argument checks and the operators' fakes on fake tensors."""
import copy
import ctypes
import warnings

import pytest
import torch
import torch.nn as nn

from fiery_b200 import _lib, install, ops  # noqa: F401
from fiery_b200.temporal import TensorCorePyramidPooling, TensorCoreTemporalBlock, aggregation_block_reason, aggregation_reason, \
    pooling_reason
from oracle import temporal_oracle as TO
from tests._temporal_models import temporal_model


def _holder(m):
    return type("M", (), {"temporal_model": m})()


def _model(rf=3, grid=(8, 8), **kw):
    torch.manual_seed(0)
    return TO.TemporalModel(70, rf, grid, start_out_channels=64, **kw)


# ------------------------------------------------------------------------------------------------------------------------------
# coverage
# ------------------------------------------------------------------------------------------------------------------------------
def test_reasons_of_the_shipped_blocks_are_none():
    for b in _model(rf=5).model:
        assert pooling_reason(b.pyramid_pooling) is None
        assert aggregation_block_reason(b) is None


@pytest.mark.parametrize("pool_sizes,needle", [([(2, 8, 8), (2, 4, 4)], "2 pool sizes"), ([(2, 4, 4)], None)])
def test_pooling_reason_pool_sizes(pool_sizes, needle):
    pp = TO.PyramidSpatioTemporalPooling(12, 4, pool_sizes)
    reason = pooling_reason(pp)
    assert (reason is None) if needle is None else (needle in reason)


def test_pooling_reason_other_windows():
    pp = TO.PyramidSpatioTemporalPooling(12, 4, [(2, 8, 8)])
    pp.features[0].avgpool = nn.AvgPool3d((2, 8, 8), stride=(1, 8, 8), padding=(1, 0, 0), count_include_pad=True)
    assert "window" in pooling_reason(pp)
    pp.features[0].avgpool = nn.AvgPool3d((2, 8, 8), stride=(1, 4, 4), padding=(1, 0, 0), count_include_pad=False)
    assert "window" in pooling_reason(pp)
    pp.features[0].avgpool = nn.MaxPool3d(2)
    assert "AvgPool3d" in pooling_reason(pp)
    assert "structure" in pooling_reason(nn.Identity())


def test_aggregation_reasons():
    assert aggregation_reason(64, [35, 35, 35], 40000) is None
    assert "129 aggregation output channels" in aggregation_reason(129, [32, 32, 32])
    assert "multiple of 4" in aggregation_reason(64, [32, 32, 32], 202)
    assert "N_out" in aggregation_reason(64, [90, 90, 90])
    b = TO.TemporalBlock(12, 8, use_pyramid_pooling=False)
    assert "no pooled channels" in aggregation_block_reason(b)
    b = TO.TemporalBlock(12, 8, use_pyramid_pooling=True, pool_sizes=[(2, 4, 4)])
    b.aggregation[0].conv = nn.Conv3d(22, 8, 1, bias=True)
    assert "bias-free 1x1x1" in aggregation_block_reason(b)
    assert "structure" in aggregation_block_reason(nn.Identity())


# ------------------------------------------------------------------------------------------------------------------------------
# install
# ------------------------------------------------------------------------------------------------------------------------------
ORDERS = [("pool", "entry", "causal"), ("entry", "causal", "pool"), ("entry", "pool", "causal"), ("pool",)]
SWAPS = {"pool": install.use_tensor_core_pyramid_pooling, "entry": install.use_tensor_core_temporal_model,
         "causal": install.use_tensor_core_causal_convs}


@pytest.mark.parametrize("order", ORDERS, ids=lambda o: "-".join(o))
@pytest.mark.parametrize("inbetween", [0, 1])
def test_swap_order_idempotence_and_state_dict(order, inbetween):
    m = temporal_model(70, 3, (8, 8), start_out_channels=64, inbetween_layers=inbetween)
    keys = list(m.state_dict())
    h = _holder(m)
    for name in order:
        SWAPS[name](h)
    blocks = [b for b in m.model if type(b).__name__ in ("TemporalBlock", "TensorCoreTemporalBlock")]
    assert len(blocks) == 2
    pps = [b.pyramid_pooling for b in blocks]
    assert all(isinstance(p, TensorCorePyramidPooling) for p in pps)
    assert all(isinstance(b, TensorCoreTemporalBlock) for b in blocks) == ("entry" in order)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        install.use_tensor_core_pyramid_pooling(h)                 # a second call does nothing
    assert [b.pyramid_pooling for b in blocks] == pps
    assert list(m.state_dict()) == keys


def test_uncovered_pooling_is_left_alone_with_one_warning():
    m = _model()
    for b in m.model:
        b.pyramid_pooling = TO.PyramidSpatioTemporalPooling(b.in_channels, b.in_channels // 3, [(2, 8, 8), (2, 4, 4)])
    install._warned.clear()
    with pytest.warns(RuntimeWarning, match="not covered by the spatial-sums kernel") as rec:
        install.use_tensor_core_pyramid_pooling(_holder(m))
    assert len(rec) == 1 and "block 0" in str(rec[0].message) and "block 1" in str(rec[0].message)
    assert all(type(b.pyramid_pooling).__name__ == "PyramidSpatioTemporalPooling" for b in m.model)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        install.use_tensor_core_pyramid_pooling(_holder(m))        # the same skip warns once


def test_identity_and_no_pyramid_models_are_left_alone():
    m = _model(use_pyramid_pooling=False)
    install.use_tensor_core_pyramid_pooling(_holder(m))
    assert not any(hasattr(b, "pyramid_pooling") for b in m.model)
    assert install.use_tensor_core_pyramid_pooling(type("M", (), {"temporal_model": nn.Identity()})()) is not None


def test_from_module_raises_on_uncovered():
    with pytest.raises(ValueError, match="2 pool sizes"):
        TensorCorePyramidPooling.from_module(TO.PyramidSpatioTemporalPooling(12, 4, [(2, 8, 8), (2, 4, 4)]))


# ------------------------------------------------------------------------------------------------------------------------------
# the pooled vector's arithmetic (means from torch on the CPU; the kernels are tested on the GPU)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [2, 3, 5])
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
def test_vector_matches_reference_pooling(s, train):
    torch.manual_seed(s)
    pp = TO.PyramidSpatioTemporalPooling(12, 4, [(2, 6, 5)]).double().train(train)
    mine = TensorCorePyramidPooling.from_module(copy.deepcopy(pp)).train(train)
    x = torch.randn(2, 12, s, 6, 5, dtype=torch.float64)
    want = pp(x)
    v = mine.vector(x.mean(dim=(3, 4)))
    got = v[..., None, None].expand(*v.shape, 6, 5)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    for (n, a), (_, b) in zip(mine.named_buffers(), pp.named_buffers()):
        assert torch.allclose(a.double(), b.double(), rtol=1e-12, atol=1e-12), n


def test_uncovered_map_runs_reference_with_one_warning():
    torch.manual_seed(0)
    pp = TO.PyramidSpatioTemporalPooling(12, 4, [(2, 4, 4)]).double()
    mine = TensorCorePyramidPooling.from_module(copy.deepcopy(pp))
    x = torch.randn(2, 12, 3, 8, 8, dtype=torch.float64)
    with pytest.warns(RuntimeWarning, match="does not cover the 8x8 map"):
        got = mine(x)
    assert torch.equal(got, pp(x))
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        mine(x)


# ------------------------------------------------------------------------------------------------------------------------------
# C ABI argument checks and fakes
# ------------------------------------------------------------------------------------------------------------------------------
def _sums_desc(b=3, c=64, s=3, pixels=40000, strides=None):
    d = _lib.SpatialSumsDesc()
    d.batch, d.channels, d.frames, d.pixels = b, c, s, pixels
    d.stride_b, d.stride_c, d.stride_t = strides or (c * s * pixels, s * pixels, pixels)
    return d


@pytest.mark.parametrize("kw,needle", [(dict(pixels=0), "pixels"), (dict(b=-1), "batch"), (dict(strides=(-4, 0, 0)), "strides")])
def test_spatial_sums_rejects(kw, needle):
    lib = _lib.load()
    assert lib.fiery_spatial_sums(_sums_desc(**kw), 256, 256, None) != 0
    assert needle in lib.fiery_last_error().decode()


def test_spatial_sums_zero_planes_is_a_no_op():
    assert _lib.load().fiery_spatial_sums(_sums_desc(s=0), None, None, None) == 0


def test_aggregation_forward_rejects():
    lib = _lib.load()
    d = _lib.TemporalEntryDesc()
    d.batch, d.frames, d.pixels, d.in_channels, d.extra_channels, d.n_segments = 3, 3, 40000, 64, 2, 3
    for i in range(3):
        d.seg_channels[i] = 35
    d.in_stride_b, d.in_stride_t, d.in_stride_c = 64 * 3 * 40000, 40000, 3 * 40000
    four = (ctypes.c_void_p * 4)(256, 256, 256, 256)
    assert lib.fiery_temporal_aggregation_forward(d, four, 256, 0, 256, None) != 0
    assert "extra_channels" in lib.fiery_last_error().decode()
    d.extra_channels, d.in_channels = 0, 129
    assert lib.fiery_temporal_aggregation_forward(d, four, 256, 0, 256, None) != 0
    assert "in_channels" in lib.fiery_last_error().decode()


def test_fakes_on_fake_tensors():
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        xf = torch.empty(2, 3, 70, 8, 8, device="cuda").permute(0, 2, 1, 3, 4)
        sums = torch.ops.fiery_b200.spatial_sums(xf)
        assert sums.shape == (2, 70, 3) and sums.dtype == torch.float32
        ps = [torch.empty(2, 35, 3, 8, 8, device="cuda", dtype=torch.float16) for _ in range(3)]
        w = torch.empty(64, 128, 1, 1, 1, device="cuda")
        v = torch.empty(2, 23, 3, device="cuda")
        z = torch.ops.fiery_b200.temporal_aggregation(ps, w, v)
        assert z.shape == (2, 64, 3, 8, 8) and z.dtype == torch.float32 and z.is_contiguous()
        g = torch.empty(2, 64, 3, 8, 8, device="cuda")
        for need in ((True, True, True), (False, True, False), (True, False, False), (False, False, True)):
            gp, gw, gv = torch.ops.fiery_b200.temporal_aggregation_backward(g, ps, w, v, *need)
            assert [tuple(t.shape) for t in gp] == ([(2, 35, 3, 8, 8)] * 3 if need[0] else [(0,)] * 3)
            assert all(t.dtype == torch.float16 for t in gp)
            assert tuple(gw.shape) == ((64, 128, 1, 1, 1) if need[1] else (0,))
            assert tuple(gv.shape) == ((2, 23, 3) if need[2] else (0,))
