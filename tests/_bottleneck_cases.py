"""Shared fixtures for the Bottleneck tests: the shapes, seeded operands, and the unfused chain of the existing entry points
(fiery_temporal_entry_*, fiery_causal_conv3d_*, fiery_batch_norm_*) that fiery_bottleneck_* must reproduce bit for bit."""
from __future__ import annotations

import ctypes

import torch

from fiery_b200 import _lib
from fiery_b200 import bottleneck as bk

# (maps, C, X, Y): every channel case of the kernels (M = C // 2 from 1 to 64, odd M, C odd), 1 and 12 maps, and grids that put a
# tile and halo edge of both 3x3 kernels (8 x 16 forward tiles, 32-column weight-gradient runs) and of the 1x1 GEMM (64 / 128-pixel
# tiles) inside or at the map's edge
SHAPES = [
    (12, 64, 200, 200),
    (1, 2, 1, 4),
    (1, 35, 7, 12),
    (12, 70, 33, 20),
    (1, 128, 33, 20),
    (3, 64, 9, 36),
    (2, 17, 8, 16),
    (1, 64, 17, 32),
    (1, 128, 400, 200),
]
SMALL = [s for s in SHAPES if s[0] * s[2] * s[3] < 100_000]


def operands(maps: int, c: int, h: int, w: int, seed: int = 0, device: str = "cuda"):
    """x (maps, C, X, Y), the three weights and the norms' 12 parameters (weight, bias, running_mean, running_var each), seeded."""
    g = torch.Generator().manual_seed(seed)
    m = c // 2
    rnd = lambda *shape, scale=1.0, off=0.0: (torch.randn(shape, generator=g) * scale + off).to(device)  # noqa: E731
    x = rnd(maps, c, h, w)
    w_d, w_c, w_u = rnd(m, c, 1, 1, scale=c ** -0.5), rnd(m, m, 3, 3, scale=(9 * m) ** -0.5), rnd(c, m, 1, 1, scale=m ** -0.5)
    norms = []
    for k in (m, m, c):
        norms += [rnd(k, scale=0.2, off=1.0), rnd(k, scale=0.2), rnd(k, scale=0.3), rnd(k, scale=0.2, off=1.0).abs() + 0.1]
    return x, (w_d, w_c, w_u), norms


def _p(t):
    return t.data_ptr() if t is not None else 0


def _call(entry, dev, *args):
    _lib.call(entry, torch.device(dev), *args)


def nan_filled(*shape, margin: int = 64, device="cuda"):
    """(view, buffer): a NaN-filled fp32 view of ``shape`` inside a buffer with ``margin`` sentinel floats on each side."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 2 * margin,), float("nan"), device=device)
    buf[:margin] = 1234.5
    buf[-margin:] = 1234.5
    return buf[margin:margin + n].view(shape), buf


def margins_intact(buf, margin: int = 64) -> bool:
    return bool((buf[:margin] == 1234.5).all() and (buf[-margin:] == 1234.5).all())


def fused_forward(x, weights, norms, training, eps=1e-5):
    """The C ABI forward into NaN-filled memory between sentinels: (out, y1, y2, y3, stats, buffers)."""
    maps, c, h, w = x.shape
    m = c // 2
    d = bk.desc(maps, h, w, c, training, eps)
    lib = _lib.load()
    packed = bk.pack_weights(list(weights))
    outs = [nan_filled(maps, c, h, w), nan_filled(maps, m, h, w), nan_filled(maps, m, h, w), nan_filled(maps, c, h, w),
            nan_filled(4 * m + 2 * c)]
    ws = _lib.workspace(lib.fiery_bottleneck_forward_workspace_bytes(d), x.device)
    ws.fill_(0xFF)
    params = [n if training is False or j % 4 < 2 else None for j, n in enumerate(norms)]
    _call("fiery_bottleneck_forward", x.device, d, x.data_ptr(), packed.data_ptr(), bk._pointers(params), outs[1][0].data_ptr(),
          outs[2][0].data_ptr(), outs[3][0].data_ptr(), outs[0][0].data_ptr(), outs[4][0].data_ptr(), ws.data_ptr())
    return [o[0] for o in outs], [o[1] for o in outs]


def fused_backward(g, x, y1, y2, y3, stats, weights, norms, training, need=(True,) * 10, eps=1e-5):
    """The C ABI backward into NaN-filled memory: ([grad_x, gW_down, gW_conv, gW_up, gw1, gb1, gw2, gb2, gw3, gb3], buffers); None
    where not asked for."""
    maps, c, h, w = x.shape
    m = c // 2
    d = bk.desc(maps, h, w, c, training, eps)
    lib = _lib.load()
    packed = bk.pack_weights(list(weights))
    shapes = [(maps, c, h, w)] + [tuple(wt.shape) for wt in weights] + [(m,), (m,), (m,), (m,), (c,), (c,)]
    outs = [nan_filled(*s) if nd else (None, None) for s, nd in zip(shapes, need)]
    ws = _lib.workspace(lib.fiery_bottleneck_backward_workspace_bytes(d), x.device)
    ws.fill_(0xFF)
    gn = [o[0] for o in outs[4:]]
    _call("fiery_bottleneck_backward", x.device, d, g.data_ptr(), x.data_ptr(), y1.data_ptr(), y2.data_ptr(), y3.data_ptr(),
          stats.data_ptr(), packed.data_ptr(), bk._pointers(norms), _p(outs[0][0]), _p(outs[1][0]), _p(outs[2][0]), _p(outs[3][0]),
          bk._pointers(gn), ws.data_ptr())
    return [o[0] for o in outs], [o[1] for o in outs if o[1] is not None]


# ------------------------------------------------------------------------------------------------------------------------------
# the unfused chain of today's entry points
# ------------------------------------------------------------------------------------------------------------------------------
def _entry_desc(maps, k, n_out, p):
    d = _lib.TemporalEntryDesc()
    d.batch, d.frames, d.pixels, d.in_channels, d.extra_channels, d.n_segments = maps, 1, p, k, 0, 1
    d.seg_channels[0] = n_out
    d.in_stride_b = d.in_stride_t = k * p
    d.in_stride_c = p
    return d


def _entry_pack(d, w2d):
    out = torch.empty(int(_lib.load().fiery_temporal_entry_packed_bytes(d)), dtype=torch.uint8, device=w2d.device)
    _call("fiery_temporal_entry_pack_weights", w2d.device, d, w2d.contiguous().data_ptr(), out.data_ptr())
    return out


def _entry_fwd(d, x, packed, n_out):
    y = torch.empty((d.batch, n_out) + tuple(x.shape[2:]), device=x.device)
    ptrs = (ctypes.c_void_p * 1)(y.data_ptr())
    _call("fiery_temporal_entry_forward", x.device, d, x.data_ptr(), 0, packed.data_ptr(), ptrs)
    return y


def _entry_dgrad(d, gy, packed, k):
    gx = torch.empty((d.batch, k) + tuple(gy.shape[2:]), device=gy.device)
    ptrs = (ctypes.c_void_p * 1)(gy.data_ptr())
    _call("fiery_temporal_entry_backward_data", gy.device, d, ptrs, packed.data_ptr(), gx.data_ptr())
    return gx


def _entry_wgrad(d, x, gy, n_out, k):
    gw = torch.empty((n_out, k), device=x.device)
    ws = _lib.workspace(_lib.load().fiery_temporal_entry_backward_weight_workspace_bytes(d), x.device)
    ptrs = (ctypes.c_void_p * 1)(gy.data_ptr())
    _call("fiery_temporal_entry_backward_weight", x.device, d, x.data_ptr(), 0, ptrs, gw.data_ptr(), ws.data_ptr())
    return gw


def _conv_desc(maps, m, h, w):
    d = _lib.CausalConv3dDesc()
    d.batch, d.frames, d.grid_x, d.grid_y, d.in_channels, d.out_channels, d.kt = maps, 1, h, w, m, m, 1
    return d


def _bn_desc(x, training, eps):
    n, c, h, w = x.shape
    d = _lib.BatchNormDesc()
    d.batch, d.channels, d.frames, d.pixels = n, c, 1, h * w
    d.stride_b, d.stride_c, d.stride_t = c * h * w, h * w, h * w
    d.training, d.relu, d.eps = int(training), 1, float(eps)
    return d


def _bn_fwd(x, p, training, eps, residual=None):
    c = x.shape[1]
    d = _bn_desc(x, training, eps)
    y, mean, var = torch.empty_like(x), torch.empty(c, device=x.device), torch.empty(c, device=x.device)
    ws = _lib.workspace(_lib.load().fiery_batch_norm_workspace_bytes(d), x.device)
    _call("fiery_batch_norm_forward", x.device, d, x.data_ptr(), _p(p[0]), _p(p[1]), _p(p[2]) if not training else 0,
          _p(p[3]) if not training else 0, _p(residual), y.data_ptr(), mean.data_ptr(), var.data_ptr(), ws.data_ptr())
    return y, mean, var


def _bn_bwd(x, g, p, mean, var, training, eps):
    c = x.shape[1]
    d = _bn_desc(x, training, eps)
    dx, dw, db = torch.empty_like(x), torch.empty(c, device=x.device), torch.empty(c, device=x.device)
    ws = _lib.workspace(_lib.load().fiery_batch_norm_workspace_bytes(d), x.device)
    _call("fiery_batch_norm_backward", x.device, d, x.data_ptr(), g.data_ptr(), _p(p[0]), _p(p[1]), mean.data_ptr(), var.data_ptr(),
          dx.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr())
    return dx, dw, db


def unfused(x, weights, norms, training, g=None, eps=1e-5):
    """The chain of today's entry points: dict of y1, y2, y3, out, stats and, with g, every gradient (dx = entry dgrad + g)."""
    maps, c, h, w = x.shape
    m, p = c // 2, h * w
    w_d, w_c, w_u = weights
    dd, du = _entry_desc(maps, c, m, p), _entry_desc(maps, m, c, p)
    pd, pu = _entry_pack(dd, w_d.reshape(m, c)), _entry_pack(du, w_u.reshape(c, m))
    cd = _conv_desc(maps, m, h, w)
    pc = torch.empty(int(_lib.load().fiery_causal_conv3d_packed_bytes(cd)), dtype=torch.uint8, device=x.device)
    _call("fiery_causal_conv3d_pack_weights", x.device, cd, w_c.contiguous().data_ptr(), pc.data_ptr())
    n1, n2, n3 = norms[0:4], norms[4:8], norms[8:12]
    r = {}
    r["y1"] = _entry_fwd(dd, x, pd, m)
    a1, m1, v1 = _bn_fwd(r["y1"], n1, training, eps)
    r["y2"] = torch.empty_like(r["y1"])
    _call("fiery_causal_conv3d_forward", x.device, cd, a1.data_ptr(), pc.data_ptr(), r["y2"].data_ptr())
    a2, m2, v2 = _bn_fwd(r["y2"], n2, training, eps)
    r["y3"] = _entry_fwd(du, a2, pu, c)
    r["out"], m3, v3 = _bn_fwd(r["y3"], n3, training, eps, residual=x)
    r["stats"] = torch.cat([m1, v1, m2, v2, m3, v3])
    if g is None:
        return r
    dy3, r["gw3"], r["gb3"] = _bn_bwd(r["y3"], g, n3, m3, v3, training, eps)
    r["gW_up"] = _entry_wgrad(du, a2, dy3, c, m).view(c, m, 1, 1)
    da2 = _entry_dgrad(du, dy3, pu, m)
    dy2, r["gw2"], r["gb2"] = _bn_bwd(r["y2"], da2, n2, m2, v2, training, eps)
    r["gW_conv"] = torch.empty_like(w_c)
    ws = _lib.workspace(_lib.load().fiery_causal_conv3d_backward_weight_workspace_bytes(cd), x.device)
    _call("fiery_causal_conv3d_backward_weight", x.device, cd, a1.data_ptr(), dy2.data_ptr(), r["gW_conv"].data_ptr(), ws.data_ptr())
    da1 = torch.empty_like(dy2)
    _call("fiery_causal_conv3d_backward_data", x.device, cd, dy2.data_ptr(), pc.data_ptr(), da1.data_ptr())
    dy1, r["gw1"], r["gb1"] = _bn_bwd(r["y1"], da1, n1, m1, v1, training, eps)
    r["gW_down"] = _entry_wgrad(dd, x, dy1, m, c).view(m, c, 1, 1)
    r["dx"] = _entry_dgrad(dd, dy1, pd, c) + g
    return r


GRAD_KEYS = ["dx", "gW_down", "gW_conv", "gW_up", "gw1", "gb1", "gw2", "gb2", "gw3", "gb3"]
