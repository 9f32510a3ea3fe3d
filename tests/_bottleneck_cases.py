"""Shared fixtures for the Bottleneck tests: the shapes, seeded operands, and the unfused chain of the existing entry points
(fiery_temporal_entry_*, fiery_causal_conv3d_*, fiery_batch_norm_*) that fiery_bottleneck_* must reproduce bit for bit; and the
envelope table with a stage-by-stage fp64 restatement of the forward and its adjoint, each element with an error bound, as
tests/_spatial_gru_cases.py does for the SpatialGRU (plain torch on any device)."""
from __future__ import annotations

import ctypes
import math

import torch
import torch.nn.functional as F

from fiery_b200 import _lib
from fiery_b200 import bottleneck as bk
from tests import _spatial_gru_cases as gc
from tests._batch_norm_cases import fmaf_exact, scale_shift

SUM, RNA, RZ, BN_SUM, ELEM = gc.SUM, gc.RNA, gc.RZ, gc.BN_SUM, gc.ELEM

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


# ------------------------------------------------------------------------------------------------------------------------------
# the envelope: a shape list reaching every kernel instantiation and tile edge, and a stage-by-stage fp64 restatement with bounds
# ------------------------------------------------------------------------------------------------------------------------------
# (maps, C, X, Y).  M = C // 2 runs over both ends of every 3x3 width N = round8(M) (M = 1, 8, 9, 16, 17, 24, 25, 32, 33, 41, 48, 49,
# 56, 57, 64), C over both sides of 64 (the up projection's and the down projection's input gradient's second 64-row block), odd C;
# X over the 8-row 3x3 tile (1, 7, 8, 9, 17), Y over the 16-column tile, 28-column halo, 32-pixel weight-gradient run and 44-column x
# run (4, 12, 16, 20, 32, 36, 132), X * Y over the 1x1 kernels' 64 / 128-pixel tiles and the batch norm's 4096-pixel pieces (4096,
# 4160, and under 32); 300 one-row maps give 300 weight-gradient tiles over 128 chunks; and the shipped shape.
ENVELOPE = [
    (2, 2, 1, 4),
    (3, 3, 1, 4),
    (3, 17, 7, 4),
    (2, 18, 8, 16),
    (1, 33, 9, 12),
    (2, 35, 17, 20),
    (1, 48, 7, 36),
    (2, 51, 9, 32),
    (1, 64, 64, 64),
    (1, 66, 65, 64),
    (2, 82, 8, 132),
    (1, 96, 17, 16),
    (2, 98, 9, 20),
    (1, 112, 7, 12),
    (1, 115, 8, 36),
    (2, 128, 9, 32),
    (300, 16, 1, 4),
    (12, 64, 200, 200),
]

WG_MAX_CHUNKS = 128             # csrc/wgrad_chunks.cuh


def _round(v, k):
    return -(-v // k) * k


def instantiations(maps, c, h, w):
    """the kernels a Bottleneck call of this shape launches, as (kernel, template argument), from the launch rules of
    csrc/causal_conv.cu and csrc/temporal_entry.cu"""
    m = c // 2
    return {("bottleneck_conv_fwd_kernel", _round(m, 8)), ("bottleneck_conv_wgrad_kernel", _round(m, 8)),
            ("bottleneck_entry_fwd_kernel", _round(_round(c, 8), 64) // 64), ("bottleneck_entry_dgrad_kernel", _round(_round(c, 32), 64) // 64),
            ("bottleneck_entry_wgrad_kernel", _round(m, 64) // 64)}


def wgrad_tiles(maps, h, w):
    """(the 3x3 weight gradient's 32-pixel run tiles, the 1x1 weight gradients' 64-pixel tiles)"""
    return maps * h * (-(-w // 32)), maps * (-(-(h * w) // 64))


def entry_wgrad_depth(maps, h, w):
    """terms along the 1x1 weight gradient's longest sum path: a chunk's 64-pixel tiles, then the chunks"""
    tiles = wgrad_tiles(maps, h, w)[1]
    chunks = min(tiles, WG_MAX_CHUNKS)
    return -(-tiles // chunks) * 64 + chunks + 8


def fmaf(a, y, c):
    """fmaf(a, y, c) rounded once to fp32, in fp64 on y's device (a, c broadcast): the fp64 sum of the exact product is right except on
    an fp32 midpoint, where _batch_norm_cases.fmaf_exact settles the few such elements on the host"""
    a, y, c = torch.broadcast_tensors(a.double(), y.double(), c.double())
    s = a * y + c
    r = s.float().double()
    o = torch.nextafter(r.float(), torch.where(r < s, torch.full_like(r, math.inf), torch.full_like(r, -math.inf)).float()).double()
    tie = torch.isfinite(s) & (s != r) & (2 * s == r + o)
    if bool(tie.any()):
        idx = tie.nonzero(as_tuple=True)
        fixed = fmaf_exact(a[idx].cpu().numpy(), y[idx].cpu().numpy(), c[idx].cpu().numpy())
        r = r.clone()
        r[idx] = torch.from_numpy(fixed).double().to(r.device)
    return r


def _ch(v):
    return v.view(1, -1, 1, 1)


def _mm(w, x):
    """the 1x1 convolution w (O, K, 1, 1) on x (n, K, X, Y)"""
    return torch.einsum("ok,nkp->nop", w.reshape(w.shape[0], -1), x.flatten(2)).view(x.shape[0], w.shape[0], *x.shape[2:])


def _mm_w(x, g):
    """the 1x1 convolution's weight gradient (O, K, 1, 1) of x (n, K, X, Y) and g (n, O, X, Y)"""
    return torch.einsum("nop,nkp->ok", g.flatten(2), x.flatten(2)).view(g.shape[1], x.shape[1], 1, 1)


def _coef(w, b, mean, var, eps, device):
    """(scale, shift uncontracted, shift contracted) (C,) fp64 from fp32 statistics: _batch_norm_cases.scale_shift"""
    f = lambda t: None if t is None else t.detach().float().cpu().numpy()    # noqa: E731
    return tuple(torch.from_numpy(v).double().to(device) for v in scale_shift(f(w), f(b), f(mean), f(var), eps))


def _relu(v):
    return torch.where(v < 0, torch.zeros_like(v), v)         # a NaN passes, as bn_relu_apply's


DEFECTS = {
    "pad_prologue": "the BN + ReLU prologue applied to the 3x3's zero fill",
    "wgrad_halo": "the prologue applied to the 3x3 weight gradient's zero-filled halo",
    "lo_hi": "the coefficients of channel c and c + 4 swapped in the 3x3's prologue",
    "rz_3x3": "the 3x3's activations truncated instead of rounded to nearest",
    "rna_1x1": "the up projection's activations rounded to nearest instead of truncated",
    "skip_before_relu": "the skip added before bn3's ReLU",
    "skip_dropped": "the skip dropped",
    "bn1_for_bn2": "bn1's coefficients used for bn2",
    "tap_dropped": "one 3x3 tap dropped",
    "run_dropped": "one 32-pixel run dropped from the 3x3 weight gradient",
    "unbiased_var": "the unbiased variance used to normalize",
}


def forward(x, weights, norms, training, eps, rounding=True, kernel=None, defect=None):
    """The Bottleneck's forward stage by stage in x's dtype (each BN + ReLU an exact fmaf in either dtype).  x (maps, C, X, Y); weights
    (W_down, W_conv, W_up); norms: the 12 of ``operands`` (weight / bias may be None; running_* read in eval).  kernel (optional): a
    run's y1, y2, y3, out and stats, fed to each stage in place of the restatement's own, so no ReLU mask can differ from the run's.
    rounding False: the module's exact math (no TF32).  defect: a key of DEFECTS, computing what a kernel with that bug would.

    Returns {"value": y1, y2, y3, out, mean1, var1, mean2, var2, mean3, var3, "bound": the same keys, and what the adjoint needs}."""
    R = gc.tf32_rna if rounding else (lambda t: t)
    Z = gc.tf32_rz if rounding else (lambda t: t)
    R3 = gc.tf32_rz if rounding and defect == "rz_3x3" else R
    Z1 = gc.tf32_rna if rounding and defect == "rna_1x1" else Z
    dt, dev = x.dtype, x.device
    maps, c, h, w = x.shape
    m = c // 2
    wd, wc, wu = (R(t.to(dt)) for t in weights)
    if defect == "tap_dropped":
        wc = wc.clone()
        wc[:, :, 0, 2] = 0
    val, bnd = {}, {}

    def norm(i, y):
        """records y's statistics and bounds; returns the exact BN + ReLU of y from the run's statistics when given: (a with the
        contracted shift, a with the other, pre, (scale, shift, mean, var))"""
        wt, bs, rm, rv = norms[4 * i:4 * i + 4]
        if training:
            mean = y.mean((0, 2, 3))
            var = y.var((0, 2, 3), unbiased=False)
            em = BN_SUM * SUM * y.abs().mean((0, 2, 3))
            ev = 2 * BN_SUM * SUM * var + 4 * em * (y - _ch(mean)).abs().mean((0, 2, 3)) + em ** 2
            if defect == "unbiased_var":
                var = y.var((0, 2, 3), unbiased=True)
        else:
            mean, var = rm.to(dt), rv.to(dt)
            em = ev = torch.zeros_like(mean)
        val[f"mean{i + 1}"], val[f"var{i + 1}"], bnd[f"mean{i + 1}"], bnd[f"var{i + 1}"] = mean, var, em, ev
        if kernel is not None:
            k = kernel["stats"].to(dt)
            o = (0, 2 * m, 4 * m)[i]
            mean, var = k[o:o + y.shape[1]], k[o + y.shape[1]:o + 2 * y.shape[1]]
        if not rounding:
            s = (wt.double() if wt is not None else 1.0) / torch.sqrt(var.double() + eps)
            sh = (bs.double() if bs is not None else 0.0) - mean.double() * s
            pre = _ch(s) * y.double() + _ch(sh)
            return _relu(pre).to(dt), _relu(pre).to(dt), pre.to(dt), (s, sh, mean, var)
        s, sh_u, sh_c = _coef(wt, bs, mean, var, eps, dev)
        if defect == "lo_hi" and i == 0:
            perm = torch.tensor([j ^ 4 if (j ^ 4) < len(s) else j for j in range(len(s))], device=dev)
            s, sh_u, sh_c = s[perm], sh_u[perm], sh_c[perm]
        pre = fmaf(_ch(s), y, _ch(sh_c))
        return _relu(pre).to(dt), _relu(fmaf(_ch(s), y, _ch(sh_u))).to(dt), pre.to(dt), (s, sh_c, mean, var)

    xz = Z(x)
    y1 = _mm(wd, xz)
    val["y1"], bnd["y1"] = y1, (c + 2) * SUM * _mm(wd.abs(), xz.abs())
    y1k = kernel["y1"].to(dt) if kernel is not None else y1
    a1, a1u, pre1, co1 = norm(0, y1k)
    a1r = R3(a1)
    if defect == "pad_prologue":
        fill = _relu(co1[1]).to(dt)
        xp = _ch(fill).expand(maps, m, h + 2, w + 2).clone()
        xp[:, :, 1:-1, 1:-1] = a1r
        y2 = F.conv2d(xp, wc)
    else:
        y2 = gc.conv(a1r, wc)
    amb1 = (R(a1u) - a1r).abs()
    val["y2"] = y2
    bnd["y2"] = (9 * m + 2) * SUM * gc.conv(a1r.abs(), wc.abs()) + gc.conv(amb1, wc.abs())
    y2k = kernel["y2"].to(dt) if kernel is not None else y2
    if defect == "bn1_for_bn2":
        n2 = norm(1, y2k)                                   # the statistics of y2 still recorded
        s, _, sh_c = _coef(norms[0], norms[1], co1[2], co1[3], eps, dev)
        pre2 = fmaf(_ch(s), y2k, _ch(sh_c)).to(dt)
        a2, a2u, co2 = _relu(pre2), _relu(pre2), n2[3]
    else:
        a2, a2u, pre2, co2 = norm(1, y2k)
    a2z = Z1(a2)
    y3 = _mm(wu, a2z)
    val["y3"] = y3
    bnd["y3"] = (m + 2) * SUM * _mm(wu.abs(), a2z.abs()) + _mm(wu.abs(), (Z1(a2u) - a2z).abs())
    y3k = kernel["y3"].to(dt) if kernel is not None else y3
    _, _, pre3, co3 = norm(2, y3k)
    wt, bs = norms[8], norms[9]
    if rounding:                                            # one fp32 add of the two fp32 values; either shift rounding
        s, sh_u, _ = _coef(wt, bs, co3[2], co3[3], eps, dev)
        pre_u = fmaf(_ch(s), y3k, _ch(sh_u))
        out, other = ((_relu(p).float() + x.float()).to(dt) for p in (pre3, pre_u))
    else:
        out = other = _relu(pre3) + x
    if defect == "skip_before_relu":
        out = other = _relu(pre3 + x)
    elif defect == "skip_dropped":
        out = other = _relu(pre3)
    val["out"], bnd["out"] = out, (other - out).abs()
    used = {"x": x, "y": (y1k, y2k, y3k), "a1": a1, "a2": a2, "pre": (pre1, pre2, pre3), "coef": (co1, co2, co3)}
    return {"value": val, "bound": bnd, "used": used, "rounding": rounding, "shape": (maps, c, h, w)}


def adjoint(fw, weights, norms, g, training, eps, defect=None, maps_total=None):
    """The adjoint of ``forward``'s stages (as they used the run's values, when given) in g's dtype, in csrc/bottleneck.cu's order
    dy3 -> dW_up, da2 -> dy2 -> dW_conv, da1 -> dy1 -> dW_down, dx = W_down^T dy1 + g, each gradient with its absolute-value twin.
    maps_total: the whole batch's maps when ``fw`` is a slice of it (eval only: then the slices' weight gradients add up), for the
    weight gradients' reduction depth.  Returns (grads, bounds) keyed as GRAD_KEYS."""
    rounding = fw["rounding"]
    R = gc.tf32_rna if rounding else (lambda t: t)
    Z = gc.tf32_rz if rounding else (lambda t: t)
    u = fw["used"]
    maps, c, h, w = fw["shape"]
    m = c // 2
    dt = g.dtype
    wd, wc, wu = (R(t.to(dt)) for t in weights)
    x = u["x"].to(dt)

    def bn_back(i, y, dy, mdy):
        """(dx, its twin, dgamma, its twin, dbeta, its twin) of norm i from (dy, twin)"""
        s, _, mean, var = u["coef"][i]
        keep = (u["pre"][i] > 0) | torch.isnan(u["pre"][i])
        gm = torch.where(keep, dy, torch.zeros_like(dy))
        mg = torch.where(keep, mdy, torch.zeros_like(mdy))
        inv = _ch(1.0 / torch.sqrt(var.to(dt) + eps))
        xhat = (y - _ch(mean.to(dt))) * inv
        sc = _ch(s.to(dt))
        if training:
            dx = sc * (gm - gm.mean((0, 2, 3), keepdim=True) - xhat * (gm * xhat).mean((0, 2, 3), keepdim=True))
            mdx = sc.abs() * (mg + mg.mean((0, 2, 3), keepdim=True) + xhat.abs() * (mg * xhat.abs()).mean((0, 2, 3), keepdim=True))
        else:
            dx, mdx = sc * gm, sc.abs() * mg
        return dx, mdx, (gm * xhat).sum((0, 2, 3)), (mg * xhat.abs()).sum((0, 2, 3)), gm.sum((0, 2, 3)), mg.sum((0, 2, 3))

    y1, y2, y3 = (t.to(dt) for t in u["y"])
    a1r, a2z = R(u["a1"].to(dt)), Z(u["a2"].to(dt))
    grads, twins, gam = {}, {}, {}
    bnb = (BN_SUM + 8) * SUM + ELEM                                  # one batch norm's backward
    dy3, mdy3, grads["gw3"], twins["gw3"], grads["gb3"], twins["gb3"] = bn_back(2, y3, g, g.abs())
    grads["gW_up"], twins["gW_up"] = _mm_w(a2z, Z(dy3)), _mm_w(a2z.abs(), mdy3)
    da2, mda2 = _mm(wu.transpose(0, 1), dy3), _mm(wu.abs().transpose(0, 1), mdy3)
    dy2, mdy2, grads["gw2"], twins["gw2"], grads["gb2"], twins["gb2"] = bn_back(1, y2, da2, mda2)
    gy2 = Z(dy2)
    if defect == "run_dropped":
        gy2 = gy2.clone()
        gy2[0, :, 0, :32] = 0
    if defect == "wgrad_halo":
        fill = _relu(u["coef"][0][1]).to(dt)
        xp = _ch(fill).expand(maps, m, h + 2, w + 2).clone()
        xp[:, :, 1:-1, 1:-1] = a1r
        cols = F.unfold(xp, 3)
        grads["gW_conv"] = torch.einsum("nop,nkp->ok", gy2.flatten(2), cols).view(m, m, 3, 3)
    else:
        grads["gW_conv"] = gc.conv_w(a1r, gy2)
    twins["gW_conv"] = gc.conv_w(a1r.abs(), mdy2)
    da1, mda1 = gc.conv_t(dy2, wc), gc.conv_t(mdy2, wc.abs())
    dy1, mdy1, grads["gw1"], twins["gw1"], grads["gb1"], twins["gb1"] = bn_back(0, y1, da1, mda1)
    xz = Z(x)
    grads["gW_down"], twins["gW_down"] = _mm_w(xz, Z(dy1)), _mm_w(xz.abs(), mdy1)
    grads["dx"] = _mm(wd.transpose(0, 1), dy1) + g
    twins["dx"] = _mm(wd.abs().transpose(0, 1), mdy1) + g.abs()
    # gamma along each gradient's longest path: a batch norm's backward, an n-term sum, and RZ for each gradient operand the tensor core
    # truncates (the run's gradient, not the restatement's, is truncated); the weights and forward activations are rounded as the
    # kernels round them, so they add nothing
    g3 = bnb
    g2 = g3 + RZ + (c + 2) * SUM + bnb
    g1 = g2 + RZ + (9 * m + 2) * SUM + bnb
    mt = maps_total or maps
    d1, d3 = entry_wgrad_depth(mt, h, w) * SUM, gc.wgrad_depth(mt, 1, h, w) * SUM
    pieces = (mt * (-(-(h * w) // 4096)) + BN_SUM + 8) * SUM
    gam = {"gw3": g3 + pieces, "gb3": g3 + pieces, "gW_up": g3 + RZ + d1, "gw2": g2 + pieces, "gb2": g2 + pieces,
           "gW_conv": g2 + RZ + d3, "gw1": g1 + pieces, "gb1": g1 + pieces, "gW_down": g1 + RZ + d1,
           "dx": g1 + RZ + (m + 2) * SUM + ELEM}
    for i, k in enumerate(("gw1", "gb1", "gw2", "gb2", "gw3", "gb3")):
        if norms[4 * (i // 2) + i % 2] is None:
            grads[k] = twins[k] = None
    bounds = {k: (gam[k] * twins[k] if twins[k] is not None else None) for k in grads}
    return grads, bounds


STAGES = ("y1", "y2", "y3", "out", "mean1", "var1", "mean2", "var2", "mean3", "var3")


def as_run(out, y1, y2, y3, stats):
    return {"out": out, "y1": y1, "y2": y2, "y3": y3, "stats": stats}


def stage_ratios(run, x, weights, norms, training, eps, dtype=torch.float64):
    """{stage: (largest err / bound, non-finite elements agree)} of a run (``as_run``) against the fp64 restatement fed the run's own
    stage inputs, and that restatement"""
    k = {n: t.to(dtype) for n, t in run.items()}
    nd = [t.to(dtype) if t is not None else None for t in norms]
    fw = forward(x.to(dtype), weights, nd, training, eps, True, k)
    m = x.shape[1] // 2
    st = k["stats"]
    got = {"y1": k["y1"], "y2": k["y2"], "y3": k["y3"], "out": k["out"]}
    for i, (o, n) in enumerate(((0, m), (2 * m, m), (4 * m, x.shape[1]))):
        got[f"mean{i + 1}"], got[f"var{i + 1}"] = st[o:o + n], st[o + n:o + 2 * n]
    return {s: gc.excess(got[s], fw["value"][s], fw["bound"][s]) for s in STAGES}, fw


def grad_ratios(fw, grads, weights, norms, g, training, eps, dtype=torch.float64):
    """{gradient: (largest err / bound, non-finite elements agree)} of ``grads`` (GRAD_KEYS order, None where not computed) against
    the fp64 adjoint of ``stage_ratios``' restatement"""
    nd = [t.to(dtype) if t is not None else None for t in norms]
    want, bound = adjoint(fw, weights, nd, g.to(dtype), training, eps)
    return {n: gc.excess(got.reshape(want[n].shape), want[n], bound[n]) for n, got in zip(GRAD_KEYS, grads)
            if got is not None and want[n] is not None}
