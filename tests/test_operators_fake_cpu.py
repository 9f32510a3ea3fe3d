"""CPU: the size rule behind the lift operator's fake plan (fiery_b200/lift.py: _plan_bytes) against the library's own
fiery_lift_plan_bytes, and the fake traced with symbolic shapes.  torch.compile sizes the plan that LiftSplat.forward makes for the
backward from this rule alone, so it must agree with the library at every frame count, camera count, feature width and grid -- and
stay an expression of the symbolic batch, or every batch size would compile its own graph."""
import pytest
import torch
from torch.fx.experimental.proxy_tensor import make_fx

from fiery_b200 import _lib, ops
from fiery_b200.lift import LiftSplat, _plan_bytes
from fiery_b200.synthetic import LiftConfig

C = 64


def _lib_plan_bytes(frames, cameras, feat_w, bev):
    d = _lib.LiftDesc()
    d.n_frames, d.n_cameras, d.depth_bins, d.channels, d.feat_h, d.feat_w = frames, cameras, 48, C, 8, feat_w
    d.bev_x, d.bev_y, d.bev_z = bev[0], bev[1], 1
    return int(_lib.load().fiery_lift_plan_bytes(d))


# 51 x 49 = 2499 pillars (a frame's touched map is not a multiple of 128 bytes), 200 x 200 = 40000 (a multiple of 64, not of 128)
@pytest.mark.parametrize("bev", [(51, 49), (200, 200)], ids=["2499", "40000"])
@pytest.mark.parametrize("feat_w", [4, 12, 13, 60, 62])
@pytest.mark.parametrize("cameras", [1, 6])
@pytest.mark.parametrize("frames", [0, 1, 7])
def test_plan_bytes_match_the_library(frames, cameras, feat_w, bev):
    assert _plan_bytes(frames, cameras, feat_w, bev[0] * bev[1]) == _lib_plan_bytes(frames, cameras, feat_w, bev)


def test_plan_bytes_round_the_touched_maps_not_the_records():
    """One frame of 2499 pillars: the records end on a 128-byte boundary and the touched map takes 2560 bytes, not 2499."""
    one = _lib_plan_bytes(1, 1, 4, (51, 49))
    assert one == _plan_bytes(1, 1, 4, 0) + 2560 and _plan_bytes(1, 1, 4, 0) % 128 == 0


# the lift envelope's 51 x 49 shape: D = 7, h = 5, w = 12, 3 cameras
CFG = LiftConfig("D7", n_cameras=3, final_dim=(40, 96), x_bound=(-51.0, 51.0, 2.0), y_bound=(-49.0, 49.0, 2.0), d_bound=(4.0, 46.0, 6.0))


def _trace(make_plan, plan=None, B=7, n=2):
    """make_fx of the lift operator with symbolic shapes at (B', n) = (7, 2), on CPU tensors: only the fake implementation runs."""
    lift = LiftSplat.from_config(CFG)
    handle = ops.register_module(lift, torch.device("cpu"))
    h, w = CFG.feat_hw
    head = torch.zeros(B * n, CFG.head_channels, h, w)
    K, E = torch.zeros(B, n, 3, 3), torch.zeros(B, n, 4, 4)
    args = (head, K, E) + ((plan,) if plan is not None else ())

    def f(head, K, E, *p):
        return torch.ops.fiery_b200.lift_splat(head, K, E, p[0] if p else None, handle, make_plan)

    gm = make_fx(f, tracing_mode="symbolic")(*args)
    (out,) = [nd for nd in gm.graph.nodes if nd.op == "output"]
    bev, plan_out = out.args[0][0].meta["val"], out.args[0][1].meta["val"]
    ins = [nd.meta["val"] for nd in gm.graph.nodes if nd.op == "placeholder"]
    return lift, bev, plan_out, ins[1].shape[0].node.expr, ins[1].shape[1].node.expr


def test_fake_plan_size_is_symbolic_in_the_batch():
    lift, bev, plan, sym_b, sym_n = _trace(make_plan=True)
    X, Y = CFG.bev_hw
    size = plan.shape[0].node.expr
    assert size.free_symbols == {sym_b, sym_n}                     # not specialised to the traced (7, 2)
    for B in (1, 2, 3, 8):
        for n in (1, 6):
            assert int(size.subs({sym_b: B, sym_n: n})) == _lib_plan_bytes(B, n, CFG.feat_hw[1], (X, Y)), (B, n)
    assert plan.dtype == torch.uint8 and bev.dtype == torch.float32 and tuple(bev.shape[1:]) == (64, X, Y)


def test_fake_returns_no_plan_when_none_is_made():
    for make_plan, plan in ((False, None), (True, torch.zeros(7, dtype=torch.uint8)), (False, torch.zeros(7, dtype=torch.uint8))):
        _, _, out, _, _ = _trace(make_plan, plan)
        assert tuple(out.shape) == (0,), (make_plan, plan is not None)
