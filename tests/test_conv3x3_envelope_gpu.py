"""The spatial GRU's 3x3 convolution kernels on their own (fiery_conv3x3_*, the same packs, launches and weight-gradient blocks the GRU
runs): forward, both input-gradient segments and the weight gradient, bit-exact against fp64 on small integers (exact in TF32 and in
every fp32 partial sum), written into NaN-filled outputs between sentinel margins, the weight gradient from a NaN-filled workspace.
Channel splits are the GRU's (C_x, C_h): the gates' conv [x, h] -> [u, r] and the state conv [x, q] -> s, including C_h in 33..60,
whose gate weight gradient has a second output block narrower than 64."""
from __future__ import annotations

import pytest
import torch
import torch.nn.functional as F

from fiery_b200 import _lib
from fiery_b200.future_prediction import (conv3x3_backward_data, conv3x3_backward_weight, conv3x3_desc, conv3x3_forward,
                                          conv3x3_pack)

pytestmark = pytest.mark.gpu

SPLITS = [(32, 64), (64, 64), (1, 8), (35, 29), (64, 1), (32, 48), (64, 40)]
MARGIN = 64                                        # floats of sentinel on each side (keeps 16-byte alignment)
SENTINEL = 12345.0


def _guarded(shape):
    """(buffer, view): the view NaN-filled, MARGIN sentinels before and after it"""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 2 * MARGIN,), SENTINEL, device="cuda")
    view = buf[MARGIN:MARGIN + n].view(shape)
    view.fill_(float("nan"))
    return buf, view


def _margins_intact(buf):
    return bool((buf[:MARGIN] == SENTINEL).all() and (buf[-MARGIN:] == SENTINEL).all())


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g).float().cuda()


def _check(maps, h, w, cin, cout, seed):
    g = torch.Generator().manual_seed(seed)
    i0, i1 = cin
    o0, o1 = cout
    d = conv3x3_desc(maps, h, w, cin, cout)
    wt = _ints((o0 + o1, i0 + i1, 3, 3), -2, 2, g)
    x0, x1 = _ints((maps, i0, h, w), -3, 3, g), (_ints((maps, i1, h, w), -3, 3, g) if i1 else None)
    gy = _ints((maps, o0 + o1, h, w), -3, 3, g)
    packed = conv3x3_pack(wt, d)
    x = torch.cat([x0] + ([x1] if i1 else []), 1).double()
    want_y = F.conv2d(x, wt.double(), padding=1)
    want_gx = torch.nn.grad.conv2d_input(x.shape, wt.double(), gy.double(), padding=1)
    want_gw = torch.nn.grad.conv2d_weight(x, wt.shape, gy.double(), padding=1)

    by0, y0 = _guarded((maps, o0, h, w))
    by1, y1 = _guarded((maps, o1, h, w)) if o1 else (None, None)
    conv3x3_forward(d, x0, x1, packed, y0, y1)
    gy0, gy1 = gy[:, :o0].contiguous(), (gy[:, o0:].contiguous() if o1 else None)
    bx0, gx0 = _guarded((maps, i0, h, w))
    bx1, gx1 = _guarded((maps, i1, h, w)) if i1 else (None, None)
    conv3x3_backward_data(d, gy0, gy1, packed, gx0, gx1)
    ws = torch.full((max(int(_lib.load().fiery_conv3x3_backward_weight_workspace_bytes(d)), 16),), 255, dtype=torch.uint8, device="cuda")
    bw, gw = _guarded(tuple(wt.shape))
    conv3x3_backward_weight(d, x0, x1, gy, gw, ws)
    torch.cuda.synchronize()

    got_y = torch.cat([y0] + ([y1] if o1 else []), 1)
    got_gx = torch.cat([gx0] + ([gx1] if i1 else []), 1)
    assert torch.equal(got_y.double(), want_y), "forward"
    assert torch.equal(got_gx.double(), want_gx), "input gradient"
    assert torch.equal(gw.double(), want_gw), "weight gradient"
    for buf in (by0, by1, bx0, bx1, bw):
        if buf is not None:
            assert _margins_intact(buf)


# (maps, X, Y): a lone 1 x 4 map, ragged 7 x 12 tiles over b 3, b 3 x T 4 and b 3 x T 5 steps as maps
SMALL = [(1, 1, 4), (3, 7, 12), (12, 7, 12), (15, 7, 12)]


@pytest.mark.parametrize("grid", SMALL, ids=lambda g: "m{}_{}x{}".format(*g))
@pytest.mark.parametrize("split", SPLITS, ids=lambda s: "cx{}_ch{}".format(*s))
@pytest.mark.parametrize("conv", ["gates", "state"])
def test_small_grids(conv, split, grid):
    cx, ch = split
    cout = (ch, ch) if conv == "gates" else (ch, 0)
    _check(*grid, (cx, ch), cout, seed=cx * 100 + ch)


@pytest.mark.parametrize("case", [(3, 200, 200, 32, 64), (3, 200, 200, 64, 64), (3, 200, 200, 32, 48), (1, 400, 200, 64, 40),
                                  (1, 400, 200, 35, 29)], ids=lambda c: "m{}_{}x{}_cx{}_ch{}".format(*c))
def test_full_maps(case):
    maps, h, w, cx, ch = case
    _check(maps, h, w, (cx, ch), (ch, ch), seed=7)
    _check(maps, h, w, (cx, ch), (ch, 0), seed=8)
