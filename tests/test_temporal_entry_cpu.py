"""CPU: the temporal entry's host side -- the oracle (oracle/temporal_oracle.py) against the golden results recorded from the reference
classes (tests/golden/temporal.npz, oracle/gen_golden_temporal.py), the C ABI's shape limits and workspace rule, the install helper,
and the operators' fakes under a symbolic trace."""
import ctypes
import os
import warnings

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.fx.experimental.proxy_tensor import make_fx
from torch.fx.experimental.symbolic_shapes import ShapeEnv

from fiery_b200 import _lib, install, ops  # noqa: F401
from fiery_b200.temporal import TensorCoreTemporalBlock, backward_weight_workspace_bytes, input_strides
from oracle import temporal_oracle as TO
from tests.conftest import GOLDEN_DIR


# ------------------------------------------------------------------------------------------------------------------------------
# oracle vs golden
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "temporal.npz"))


def _oracle(name):
    return TO.TemporalModel(14, 3, (4, 4), start_out_channels=8) if name == "model" else TO.TemporalBlock(8, 8)


@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("name", ["model", "block"])
def test_oracle_matches_reference_golden(golden, name, train):
    """Identical state_dict keys; outputs, input gradient, parameter gradients and running statistics bit-equal to the reference's."""
    m = _oracle(name)
    sd_keys = [k[len(f"{name}__sd__"):] for k in golden.files if k.startswith(f"{name}__sd__")]
    assert sorted(sd_keys) == sorted(m.state_dict())
    m.load_state_dict({k: torch.from_numpy(golden[f"{name}__sd__{k}"]) for k in sd_keys})
    m.train(train)
    x = torch.from_numpy(golden[f"{name}__x"]).requires_grad_(True)
    y = m(x)
    y.backward(torch.from_numpy(golden[f"{name}__gout"]))
    tag = f"{name}__{'train' if train else 'eval'}__"
    assert np.array_equal(y.detach().numpy(), golden[tag + "y"])
    assert np.array_equal(x.grad.numpy(), golden[tag + "gx"])
    for n, p in m.named_parameters():
        assert np.array_equal(p.grad.numpy(), golden[f"{tag}grad.{n}"]), n
    for n, b in m.named_buffers():
        assert np.array_equal(b.numpy(), golden[f"{tag}buf.{n}"]), n


# ------------------------------------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------------------------------------
def _desc(b=3, s=3, pixels=40000, K=70, E=0, segs=(35, 35, 35, 64)):
    d = _lib.TemporalEntryDesc()
    d.batch, d.frames, d.pixels, d.in_channels, d.extra_channels = b, s, pixels, K, E
    d.n_segments = len(segs)
    for i, c in enumerate(segs):
        d.seg_channels[i] = c
    d.in_stride_b, d.in_stride_t, d.in_stride_c = s * K * pixels, K * pixels, pixels
    return d


def _calls(d):
    """every entry point, with non-null dummy pointers that a rejected call never touches"""
    lib, p = _lib.load(), 256
    four = (ctypes.c_void_p * 4)(p, p, p, p)
    return {
        "pack": lambda: lib.fiery_temporal_entry_pack_weights(d, p, p, None),
        "forward": lambda: lib.fiery_temporal_entry_forward(d, p, p, p, four, None),
        "backward_data": lambda: lib.fiery_temporal_entry_backward_data(d, four, p, p, None),
        "backward_weight": lambda: lib.fiery_temporal_entry_backward_weight(d, p, p, four, p, p, None),
    }


@pytest.mark.parametrize("field,kw", [("in_channels K", dict(K=129)), ("N_out", dict(segs=(64, 64, 64, 65))),
                                      ("extra_channels E", dict(E=9)), ("pixels X*Y", dict(pixels=202)),
                                      ("N_out with each segment rounded up", dict(segs=(63, 63, 63, 65)))],
                         ids=["K129", "N257", "E9", "XY%4", "Npad"])
def test_limits_are_rejected_naming_the_field(field, kw):
    d = _desc(**kw)
    for name, call in _calls(d).items():
        assert call() == -1, name
        assert field in _lib.load().fiery_last_error().decode(), name
    assert _lib.load().fiery_temporal_entry_packed_bytes(d) == 0
    assert _lib.load().fiery_temporal_entry_backward_weight_workspace_bytes(d) == 0


def test_limits_themselves_are_accepted():
    lib = _lib.load()
    assert lib.fiery_temporal_entry_packed_bytes(_desc(K=128, E=8, segs=(64, 64, 64, 64))) > 0
    assert lib.fiery_temporal_entry_backward_weight_workspace_bytes(_desc(K=1, E=0, segs=(1,), pixels=4)) > 0


@pytest.mark.parametrize("batch,frames", [(0, 3), (3, 0), (0, 0)])
def test_zero_frames_is_a_successful_no_op(batch, frames):
    d = _desc(b=batch, s=frames)
    calls = _calls(d)
    assert calls["forward"]() == 0 and calls["backward_data"]() == 0
    assert _lib.load().fiery_temporal_entry_backward_weight_workspace_bytes(d) == 0


def _workspace_rule(frames, pixels, K, E, segs):
    """128 chunks at most of 64-pixel tiles; a chunk's partial is (Npad rounded up to 64) x (K + E rounded up to 64) floats, Npad
    the segments' channel counts each rounded up to 8"""
    tiles = frames * -(-pixels // 64)
    npad = sum(-(-c // 8) * 8 for c in segs)
    return min(tiles, 128) * (-(-npad // 64) * 64) * (-(-(K + E) // 64) * 64) * 4


@pytest.mark.parametrize("b,s,grid,K,E,segs", [
    (3, 3, (200, 200), 70, 0, (35, 35, 35, 64)), (4, 3, (400, 200), 64, 6, (35, 35, 35, 64)), (3, 3, (200, 200), 64, 0, (32, 32, 32)),
    (1, 1, (2, 2), 64, 0, (32, 32, 32)), (1, 1, (8, 8), 128, 8, (64, 64, 64, 64)), (2, 3, (52, 49), 1, 0, (1,)),
    (1, 2, (320, 192), 70, 0, (35, 35, 35, 64))])
def test_workspace_rule(b, s, grid, K, E, segs):
    got = backward_weight_workspace_bytes((b, K, s, *grid), segs, E)
    assert got == _workspace_rule(b * s, grid[0] * grid[1], K, E, segs)
    assert got <= 128 * 256 * 192 * 4                               # 24 MiB at the limits


def test_input_strides():
    frame_major = torch.empty(2, 3, 70, 8, 8).permute(0, 2, 1, 3, 4)
    assert input_strides(frame_major.shape, frame_major.stride()) == frame_major.stride()
    odd = torch.empty(2, 70, 3, 8, 9)[..., :6]                       # rows not contiguous: read from a contiguous copy
    assert input_strides(odd.shape, odd.stride()) == (70 * 3 * 48, 3 * 48, 48, 6, 1)
    # expanded or overlapping dimensions would make the input gradient's writes collide: contiguous copy
    expanded = torch.empty(1, 70, 1, 8, 8).expand(2, 70, 3, 8, 8)
    assert input_strides(expanded.shape, expanded.stride()) == (70 * 3 * 64, 3 * 64, 64, 8, 1)
    overlap = torch.empty(4096).as_strided((2, 70, 3, 8, 8), (64, 4, 8, 8, 1))
    assert input_strides(overlap.shape, overlap.stride()) == (70 * 3 * 64, 3 * 64, 64, 8, 1)


# ------------------------------------------------------------------------------------------------------------------------------
# install helper
# ------------------------------------------------------------------------------------------------------------------------------
class _Fiery(torch.nn.Module):
    def __init__(self, temporal_model):
        super().__init__()
        self.temporal_model = temporal_model


class TemporalModelIdentity(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.receptive_field = 1


def test_install_swaps_covered_blocks_and_keeps_keys():
    model = _Fiery(TO.TemporalModel(70, 3, (200, 200), start_out_channels=64))
    keys = list(model.state_dict())
    params = {n: p for n, p in model.named_parameters()}
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        install.use_tensor_core_temporal_model(model)
    assert all(isinstance(b, TensorCoreTemporalBlock) for b in model.temporal_model.model)
    assert list(model.state_dict()) == keys
    assert all(p is params[n] for n, p in model.named_parameters())      # adopted, not copied
    blocks = list(model.temporal_model.model)
    install.use_tensor_core_temporal_model(model)                         # idempotent
    assert list(model.temporal_model.model) == blocks and list(model.state_dict()) == keys


def test_install_leaves_uncovered_blocks_with_one_warning():
    install._warned.clear()
    tm = TO.TemporalModel(70, 3, (5, 5), start_out_channels=64)          # 25 pixels: no 16-byte TMA pitch
    wide = TO.TemporalModel(130, 2, (8, 8), start_out_channels=64)       # K = 130
    biased = TO.TemporalModel(70, 2, (8, 8), start_out_channels=64)
    biased.model[0].convolution_paths[2].conv = torch.nn.Conv3d(70, 35, 1, bias=True)
    for m, what in ((tm, "X*Y = 25"), (wide, "K = 130"), (biased, "bias-free")):
        with pytest.warns(RuntimeWarning, match=what):
            install.use_tensor_core_temporal_model(_Fiery(m))
        assert not any(isinstance(b, TensorCoreTemporalBlock) for b in m.model)
    with warnings.catch_warnings():
        warnings.simplefilter("error")                                   # the same reasons do not warn twice
        install.use_tensor_core_temporal_model(_Fiery(tm))
    ident = _Fiery(TemporalModelIdentity())
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        assert install.use_tensor_core_temporal_model(ident) is ident


def test_block_without_pooling_on_an_uncovered_map_runs_the_reference_convs():
    """install() learns the map size only from a block's pyramid pooling; a block without one checks X*Y when it is called: a map
    the TMA cannot take (X*Y % 4 != 0) runs the block's own Conv3d, with one warning, and gives the reference block's result."""
    torch.manual_seed(0)
    ref = TO.TemporalBlock(16, 8)
    tm = TO.TemporalModel(16, 2, (5, 5), start_out_channels=8, use_pyramid_pooling=False)
    tm.model[0] = ref
    model = _Fiery(tm)
    install.use_tensor_core_temporal_model(model)
    blk = model.temporal_model.model[0]
    assert isinstance(blk, TensorCoreTemporalBlock)
    x = torch.randn(2, 16, 3, 5, 5)
    with pytest.warns(RuntimeWarning, match="X\\*Y = 25"):
        got = blk(x)
    assert torch.equal(got, TO.TemporalBlock.forward(ref, x))


def test_swapped_block_follows_sync_batchnorm_conversion():
    """Children are looked up at call time, so a conversion after the swap reaches the modules the forward uses."""
    model = _Fiery(TO.TemporalModel(70, 3, (8, 8), start_out_channels=64))
    install.use_tensor_core_temporal_model(model)
    conv = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    blk = conv.temporal_model.model[0]
    assert isinstance(blk, TensorCoreTemporalBlock)
    assert isinstance(blk.convolution_paths[0][0].norm, torch.nn.SyncBatchNorm)
    assert isinstance(blk.projection[1], torch.nn.SyncBatchNorm)


# ------------------------------------------------------------------------------------------------------------------------------
# fakes
# ------------------------------------------------------------------------------------------------------------------------------
def test_fakes_trace_symbolically():
    """The forward's fake gives each output (b, C_q, s, X, Y) contiguous, the backward's gives grad_x the input's strides when the
    kernels read it as it lies (the permuted concat) and each weight gradient its weight's shape; b and s stay symbolic."""
    def fwd_bwd(x, w0, w1, w2, w3, g0, g1, g2, g3):
        ys = torch.ops.fiery_b200.temporal_entry(x, [w0, w1, w2, w3], None)
        gx, gw = torch.ops.fiery_b200.temporal_entry_backward([g0, g1, g2, g3], x, [w0, w1, w2, w3], None, True, True)
        return ys, gx, gw

    with FakeTensorMode(shape_env=ShapeEnv()) as mode:
        base = torch.empty(3, 2, 70, 8, 8, device="cuda")
        x = base.permute(0, 2, 1, 3, 4)
        ws = [torch.empty(c, 70, 1, 1, 1, device="cuda") for c in (35, 35, 35, 64)]
        gs = [torch.empty(3, c, 2, 8, 8, device="cuda") for c in (35, 35, 35, 64)]
        gm = make_fx(fwd_bwd, tracing_mode="symbolic")(x, *ws, *gs)
        ys, gx, gw = gm(x, *ws, *gs)
    assert [tuple(y.shape) for y in ys] == [(3, c, 2, 8, 8) for c in (35, 35, 35, 64)] and all(y.is_contiguous() for y in ys)
    assert gx.stride() == x.stride()
    assert [tuple(g.shape) for g in gw] == [tuple(w.shape) for w in ws]
    assert "fiery_b200.temporal_entry" in str(gm.code) and "fiery_b200.temporal_entry_backward" in str(gm.code)
