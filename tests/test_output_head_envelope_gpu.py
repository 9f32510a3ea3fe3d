"""The output head through the C ABI across its accepted shapes: every channel case of the entry's K padding, every n from 1 to 8,
pixel counts at the 128-pixel tile and 4096-pixel piece edges, train and eval, each against the fp64 restatement; and one y past 2^31
bytes.  H100 only."""
from __future__ import annotations

import pytest
import torch

from tests import _output_head_cases as oc

pytestmark = pytest.mark.gpu

CHANNELS = (1, 8, 63, 64, 65, 128)
# (X, Y): 4 pixels, one short of / at / one past a 128-pixel tile, at / past a 4096-pixel piece
GRIDS = ((1, 4), (4, 31), (4, 32), (4, 33), (64, 64), (41, 100))
CASES = [(c, n, GRIDS[(i + n) % len(GRIDS)], (i + n) % 2 == 0) for i, c in enumerate(CHANNELS) for n in range(1, 9)]


@pytest.mark.parametrize("c,n,grid,training", CASES, ids=lambda v: str(v))
def test_envelope(c, n, grid, training):
    h, w = grid
    maps = 3
    y, w1, b1, norm = oc.operands(maps, c, n, h, w, seed=c * 10 + n)
    (out, mean, var), bufs = oc.fused_forward(y, w1, b1, norm, training)
    assert all(oc.margins_intact(b) for b in bufs)
    ratios, fw = oc.stage_ratios((out, mean, var), y, w1, b1, norm, training, 1e-5)
    assert all(same and r <= 1.0 for r, same in ratios.values()), ratios
    g = torch.randn_like(out)
    grads, bufs = oc.fused_backward(g, y, mean, var, w1, b1, norm, training)
    assert all(oc.margins_intact(b) for b in bufs)
    r = oc.grad_ratios(fw, grads, w1, b1, norm, g, training, 1e-5)
    assert all(same and v <= 1.0 for v, same in r.values()), r


def test_y_past_2_31_bytes():
    """eval: every map is independent of the others, so the last map of a > 2 GiB y must come out bit for bit as on its own"""
    maps, c, n, h, w = 19, 128, 2, 480, 480                # 2.24e9 bytes
    torch.manual_seed(0)
    y = torch.randn(maps, c, h, w, device="cuda")
    _, w1, b1, norm = oc.operands(1, c, n, 4, 4)
    (out, mean, var), _ = oc.fused_forward(y, w1, b1, norm, False)
    g = torch.randn_like(out)
    grads, _ = oc.fused_backward(g, y, mean, var, w1, b1, norm, False, need=(True, False, False, False, False))
    gy = grads[0][-1:].clone()
    del grads
    last = y[-1:].clone()
    del y
    (out1, _, _), _ = oc.fused_forward(last, w1, b1, norm, False)
    assert torch.equal(out[-1:], out1)
    g1, _ = oc.fused_backward(g[-1:].contiguous(), last, mean, var, w1, b1, norm, False, need=(True, False, False, False, False))
    assert torch.equal(gy, g1[0])
