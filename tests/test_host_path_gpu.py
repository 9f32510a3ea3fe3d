"""GPU: the weight-pack cache (fiery_b200/_lib.py: ``packed``) over training steps of a chain with every tensor-core layer swapped in:
DepthLayer -> warped lift -> temporal model (entries and causal convolutions, with an in-between Bottleneck3D) -> FirstConv."""
import collections

import pytest
import torch
import torch.nn as nn

from fiery_b200 import _lib, bev_conv, causal_conv, depth_layer, install, temporal
from fiery_b200.lift import LiftSplat
from fiery_b200.synthetic import CONFIGS, LiftConfig, make_calibration, make_egomotion
from tests._temporal_models import temporal_model

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def test_each_pack_is_made_once_per_optimizer_step(monkeypatch):
    made = collections.Counter()

    def counted(module, name):
        fn = getattr(module, name)

        def pack(weights, *args):
            ws = [weights] if isinstance(weights, torch.Tensor) else weights
            made[(name, tuple(w.data_ptr() for w in ws), args)] += 1
            return fn(weights, *args)
        monkeypatch.setattr(module, name, pack)
    for module, name in ((depth_layer, "pack_weight"), (bev_conv, "pack_weight"), (bev_conv, "pack_weight_transposed"),
                         (temporal, "pack_weights"), (causal_conv, "pack_weights")):
        counted(module, name)

    s = 3
    cfg = LiftConfig(**{**CONFIGS["cfg1_tiny"].__dict__, "frames": s, "x_bound": (-52.0, 52.0, 2.0), "y_bound": (-48.0, 48.0, 2.0)})
    grid = cfg.bev_hw
    torch.manual_seed(0)
    depth = depth_layer.DepthLayer(cfg.head_channels).to(DEV)
    lift = LiftSplat.from_config(cfg).to(DEV)
    model = temporal_model(70, s, grid, start_out_channels=64, inbetween_layers=1).to(DEV)
    holder = type("M", (), {"temporal_model": model})()
    install.use_tensor_core_temporal_model(holder)
    install.use_tensor_core_causal_convs(holder)
    first = bev_conv.FirstConv.from_conv(nn.Conv2d(64, 64, 7, stride=2, padding=3, bias=False)).to(DEV)
    params = [*depth.parameters(), *model.parameters(), *first.parameters()]
    opt = torch.optim.SGD(params, lr=1e-3)
    h, w = cfg.feat_hw
    feat = torch.randn(s * cfg.n_cameras, 128, h, w, device=DEV)
    K, E = (torch.from_numpy(a).to(DEV) for a in make_calibration(cfg, seed=1))
    flow = torch.from_numpy(make_egomotion(1, s, seed=0)).to(DEV)
    ext = (float(cfg.x_bound[1]), float(cfg.y_bound[1]))

    def step():
        opt.zero_grad()
        bev = lift.forward_warped(depth(feat), K, E, flow, ext)
        y = temporal.temporal_model_forward(model, bev, flow)
        first(y[:, 0]).square().mean().backward()
        opt.step()

    # one per DepthLayer operand dtype, two for FirstConv, three per TemporalBlock (its entry and two causal convolutions), one per
    # Bottleneck3D: here 1 + 2 + 2 * 3 + 2 * 1
    n_packs = 11
    assert n_packs <= _lib._PACK_CACHE_SIZE
    step()
    assert len(made) == n_packs and set(made.values()) == {1}, made
    step()
    assert len(made) == n_packs and set(made.values()) == {2}, made
