"""Shared fixtures for the output-head tests (fiery_output_head_*): seeded operands, the C ABI calls into NaN-filled memory, and an
fp64 restatement of the operator from the kernel's own inputs, each element with an error bound from its absolute-value twin, as
tests/_bottleneck_cases.py does for the Bottleneck (plain torch on any device)."""
from __future__ import annotations

import torch

from fiery_b200 import _lib
from fiery_b200 import decoder as dec
from tests import _spatial_gru_cases as gc
from tests._bottleneck_cases import BN_SUM, ELEM, SUM, _ch, _coef, _mm, _mm_w, _relu, fmaf, margins_intact, nan_filled  # noqa: F401

GRAD_KEYS = ("gy", "gbw", "gbb", "gW", "gb")


def operands(maps: int, c: int, n: int, h: int, w: int, seed: int = 0, device: str = "cuda"):
    """y (maps, C, X, Y), W1 (n, C, 1, 1), b1 (n,) and the norm's (weight, bias, running_mean, running_var), seeded."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *shape, scale=1.0, off=0.0: (torch.randn(shape, generator=g) * scale + off).to(device)  # noqa: E731
    y = rnd(maps, c, h, w, scale=0.5, off=0.1)
    w1, b1 = rnd(n, c, 1, 1, scale=c ** -0.5), rnd(n, scale=0.5)
    norm = [rnd(c, scale=0.2, off=1.0), rnd(c, scale=0.2), rnd(c, scale=0.3), rnd(c, scale=0.2, off=1.0).abs() + 0.1]
    return y, w1, b1, norm


def integer_operands(maps: int, c: int, n: int, h: int, w: int, seed: int = 0, device: str = "cuda"):
    """Small-integer operands for bit-exact checks: y, W1, b1 integers (exact in TF32), eval statistics with var + eps = 1/4 (scale a
    power of two), so every product and sum the kernels form is exact in fp32 whatever its order."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda lo, hi, *shape: torch.randint(lo, hi, shape, generator=g).float().to(device)  # noqa: E731
    y = ri(-4, 5, maps, c, h, w)
    w1, b1 = ri(-3, 4, n, c, 1, 1), ri(-8, 9, n)
    norm = [ri(-2, 3, c), ri(-4, 5, c), ri(-2, 3, c), torch.full((c,), 0.25, device=device)]
    return y, w1, b1, norm


def _p(t):
    return t.data_ptr() if t is not None else 0


# ------------------------------------------------------------------------------------------------------------------------------
# the envelope: a shape table, and a host model of the forward's launch (csrc/temporal_entry.cu's te_stages, csrc/common.cuh's
# persistent_grid) that shows which tile, ring and piece cases the table reaches on a device of a given SM count
# ------------------------------------------------------------------------------------------------------------------------------
# (maps, C, n, X, Y): every channel count on both sides of each K padding class edge (Kpad = 32 / 64 / 96 / 128 for C = 1..32 /
# 33..64 / 65..96 / 97..128) and C = 2 (C = 2 mod 4, so the planes are 8-byte aligned only); every n from 1 to 8 in at least two Kpad
# classes; X * Y at every class of the 128-pixel tile's last-tile split between the two consumer warpgroups (P % 128 = 4, 60: warpgroup
# 1 idle; 64: warpgroup 1 at n_valid 0; 68, 124: warpgroup 1 partial; 0: both full) and at the norm's 4096-pixel piece edges (4092,
# 4096, 4100, 8188); the minimum count of 1 map of 4 pixels; and 7 maps of 19 full tiles (133 tiles: not a multiple of the grid on
# 114 or 132 SMs).
SHAPES = [
    (1, 1, 1, 1, 4),
    (3, 2, 2, 4, 33),
    (2, 8, 3, 6, 10),
    (3, 31, 4, 8, 8),
    (2, 32, 5, 4, 17),
    (2, 33, 6, 4, 31),
    (3, 63, 7, 4, 32),
    (2, 64, 8, 4, 47),
    (2, 65, 1, 8, 24),
    (3, 96, 2, 14, 14),
    (2, 97, 3, 12, 21),
    (2, 127, 4, 16, 16),
    (2, 128, 5, 62, 66),
    (2, 2, 6, 64, 64),
    (2, 96, 7, 41, 100),
    (1, 127, 8, 89, 92),
    (7, 17, 2, 38, 64),
]
# (maps, C, n, X, Y, training): every shape in both modes
ENVELOPE = [s + (t,) for s in SHAPES for t in (True, False)]
# the shipped heads: 15 and 18 maps (3 and 6 frames of 5 / 3 samples) of the decoder's 64 x 200 x 200 output, segmentation (2) and
# center (1): 313 tiles per map, the last with 64 pixels (warpgroup 1 at n_valid 0 in every map)
SHIPPED = [(m, 64, n, 200, 200, True) for m in (15, 18) for n in (1, 2)]

SMEM_MAX, SMEM_SLACK = 232448, 1024 + 256            # csrc/temporal_entry.cu: TE_SMEM_MAX, TE_SMEM_SLACK
STG_BYTES, ROW_TABLE_BYTES = 2 * 32 * 66 * 4, 2 * 256 * (8 + 4)
COEF_BYTES = 128 * 5 * 4                             # 128 BnCoef of 5 floats
TILE_PX, PIECE_PX = 128, 4096
KPADS = (32, 64, 96, 128)


def kpad(c: int) -> int:
    return -(-c // 32) * 32


def ring_depth(c: int) -> int:
    """te_stages for output_head_fwd_kernel: the forward weights (one 64-row block of Kpad columns), two staging tiles, the row tables
    and the coefficients fixed; 128 pixels x Kpad channels per stage; at most 4"""
    k = kpad(c)
    fixed = 64 * k * 4 + STG_BYTES + ROW_TABLE_BYTES + COEF_BYTES
    return min((SMEM_MAX - SMEM_SLACK - fixed) // (4 * k * TILE_PX), 4)


def persistent_grid(n_tiles: int, sms: int) -> int:
    waves = -(-n_tiles // sms)
    return -(-n_tiles // waves)


def reach(case, sms: int) -> dict:
    """what one ENVELOPE case exercises on a device of ``sms`` SMs"""
    maps, c, n, h, w, training = case
    p = h * w
    tiles = maps * -(-p // TILE_PX)
    grid = persistent_grid(tiles, sms)
    depth = ring_depth(c)
    return {"kpad": kpad(c), "n": n, "depth": depth, "tiles": tiles, "grid": grid, "tail": p % TILE_PX,
            "wg1_valid": (p - 1) % TILE_PX + 1 - 64,      # warpgroup 1's n_valid on each map's last tile
            "min_per_cta": tiles // grid, "uneven": tiles % grid != 0,
            "ring_wrap": tiles // grid >= 2 * depth + 1,  # every CTA uses each ring stage at least twice, so every phase flips
            "frame_change": grid < tiles and -(-p // TILE_PX) < tiles, "piece_edge": p in (PIECE_PX - 4, PIECE_PX, PIECE_PX + 4, 2 * PIECE_PX - 4),
            "min_count": training and maps * p == 4}


def wrap_case(kp: int, sms: int):
    """a training case at K padding kp whose tile count makes every CTA of a ``sms``-SM device wrap its ring twice: C = kp - 2, maps
    of 100 x 130 pixels (102 tiles, the last with 72 pixels), as few maps as that takes"""
    c, n = kp - 2, {32: 8, 64: 3, 96: 5, 128: 2}[kp]
    maps = 1
    while not reach((maps, c, n, 100, 130, True), sms)["ring_wrap"]:
        maps += 1
    return (maps, c, n, 100, 130, True)


def fused_forward(y, w1, b1, norm, training, eps=1e-5):
    """The C ABI forward into NaN-filled memory between sentinels: ([out, mean, var], buffers)."""
    maps, c, h, w = y.shape
    n = w1.shape[0]
    d = dec.desc(maps, h, w, c, n, training, eps)
    packed = dec.pack_weights([w1, b1])
    outs = [nan_filled(maps, n, h, w), nan_filled(c), nan_filled(c)]
    ws = _lib.workspace(_lib.load().fiery_output_head_forward_workspace_bytes(d), y.device)
    ws.fill_(0xFF)
    rm, rv = (None, None) if training else (norm[2], norm[3])
    _lib.call("fiery_output_head_forward", y.device, d, y.data_ptr(), packed.data_ptr(), _p(norm[0]), _p(norm[1]), _p(rm), _p(rv),
              outs[0][0].data_ptr(), outs[1][0].data_ptr(), outs[2][0].data_ptr(), ws.data_ptr())
    return [o[0] for o in outs], [o[1] for o in outs]


def fused_backward(g, y, mean, var, w1, b1, norm, training, need=(True,) * 5, eps=1e-5, ws=None):
    """The C ABI backward into NaN-filled memory: ([grad_y, grad_bn_weight, grad_bn_bias, grad_W1 (n, C), grad_b1], buffers); None
    where not asked for.  ws: a workspace to use (else a fresh 0xFF-filled one)."""
    maps, c, h, w = y.shape
    n = w1.shape[0]
    d = dec.desc(maps, h, w, c, n, training, eps)
    shapes = [(maps, c, h, w), (c,), (c,), (n, c), (n,)]
    outs = [nan_filled(*s) if nd else (None, None) for s, nd in zip(shapes, need)]
    if ws is None:
        ws = _lib.workspace(_lib.load().fiery_output_head_backward_workspace_bytes(d), y.device)
        ws.fill_(0xFF)
    _lib.call("fiery_output_head_backward", y.device, d, g.data_ptr(), y.data_ptr(), mean.data_ptr(), var.data_ptr(), w1.contiguous().data_ptr(),
              _p(norm[0]), _p(norm[1]), *(_p(o[0]) for o in outs), ws.data_ptr())
    return [o[0] for o in outs], [o[1] for o in outs if o[1] is not None]


# ------------------------------------------------------------------------------------------------------------------------------
# the fp64 restatement
# ------------------------------------------------------------------------------------------------------------------------------
DEFECTS = {
    "w1_transposed": "W1 read with its two strides swapped",
    "mask_side": "the ReLU mask taken from the wrong side of 0",
    "bias_grad_dropped": "the bias gradient dropped",
    "batch_stats_in_eval": "the batch statistics used in eval",
    "unbiased_var": "the unbiased variance used to normalize",
    "da_wrong_operand": "da summed over the forward's output instead of grad_out",
    "b1_tf32": "b1 rounded to TF32 like W1",
    "da_packed_w1": "da formed with the packed (TF32-rounded) W1 instead of the fp32 one",
    "dw1_rz_a": "dW1 formed from the truncated a the tensor core reads",
    "a_rna": "a rounded to nearest instead of truncated",
    "eps_outside_sqrt": "eps added outside the square root: weight / (sqrt(var) + eps)",
    "db1_all_channels": "db1 summed over every channel's pieces instead of channel 0's",
}
# the defects that change the forward (the others change only the adjoint); and the module-level one (``running_update``)
FORWARD_DEFECTS = ("w1_transposed", "unbiased_var", "batch_stats_in_eval", "b1_tf32", "a_rna", "eps_outside_sqrt")
MODULE_DEFECTS = {"running_var_biased": "the running variance moved toward the biased batch variance"}


def _w1(w1, dt, rounding, defect=None):
    n, c = w1.shape[0], w1.shape[1]
    w = w1.to(dt).reshape(n, c)
    if defect == "w1_transposed":
        w = w.flatten().view(c, n).t()
    return gc.tf32_rna(w) if rounding else w


def forward(y, w1, b1, norm, training, eps, rounding=True, kernel=None, defect=None):
    """The operator in y's dtype: k = bn's coefficients (training: y's batch statistics; eval: the running ones), a = relu(fmaf(scale, y,
    shift)), out = rna(W1) rz(a) + b1.  kernel (optional): a run's (mean, var), used for the coefficients so no ReLU mask can differ
    from the run's.  rounding False: the module's exact math (no TF32, shift in fp64 without the fmaf).  defect: a key of DEFECTS.
    Returns {"value": out, mean, var, "bound": the same keys, and what the adjoint needs}."""
    dt = y.dtype
    wt, bs, rm, rv = norm
    if training or defect == "batch_stats_in_eval":
        mean = y.mean((0, 2, 3))
        var = y.var((0, 2, 3), unbiased=defect == "unbiased_var")
        em = BN_SUM * SUM * y.abs().mean((0, 2, 3))
        ev = 2 * BN_SUM * SUM * var + 4 * em * (y - _ch(mean)).abs().mean((0, 2, 3)) + em ** 2
    else:
        mean, var = rm.to(dt), rv.to(dt)
        em = ev = torch.zeros_like(mean)
    val, bnd = {"mean": mean, "var": var}, {"mean": em, "var": ev}
    if kernel is not None:
        mean, var = kernel[0].to(dt), kernel[1].to(dt)
    if rounding and defect == "eps_outside_sqrt":
        w64 = wt.double() if wt is not None else torch.ones_like(mean.double())
        s = (w64 / (torch.sqrt(var.double()) + eps)).float().double()
        sh_u = sh_c = ((bs.double() if bs is not None else 0.0) - mean.double() * s).float().double()
        pre = fmaf(_ch(s), y, _ch(sh_c)).to(dt)
        a, a_u = _relu(pre), _relu(pre)
    elif rounding:
        s, sh_u, sh_c = _coef(wt, bs, mean, var, eps, y.device)
        pre = fmaf(_ch(s), y, _ch(sh_c)).to(dt)
        a, a_u = _relu(pre), _relu(fmaf(_ch(s), y, _ch(sh_u))).to(dt)
    else:
        s = (wt.to(dt) if wt is not None else 1.0) / torch.sqrt(var.to(dt) + eps)
        sh = (bs.to(dt) if bs is not None else 0.0) - mean.to(dt) * s
        pre = _ch(s) * y + _ch(sh)
        a = a_u = _relu(pre)
    W = _w1(w1, dt, rounding, defect)
    Z = gc.tf32_rz if rounding else (lambda t: t)
    if rounding and defect == "a_rna":
        Z = gc.tf32_rna
    az = Z(a)
    bb = gc.tf32_rna(b1.to(dt)) if defect == "b1_tf32" else b1.to(dt)
    out = _mm(W.view(*W.shape, 1, 1), az) + _ch(bb)
    c = y.shape[1]
    bnd["out"] = (c + 3) * SUM * (_mm(W.abs().view(*W.shape, 1, 1), az.abs()) + _ch(b1.to(dt).abs())) + \
        _mm(W.abs().view(*W.shape, 1, 1), (Z(a_u) - az).abs())
    val["out"] = out
    used = {"y": y, "a": a, "pre": pre, "s": s, "mean": mean, "var": var}
    return {"value": val, "bound": bnd, "used": used, "rounding": rounding}


def _masked_da(fw, w1, g, eps, defect=None):
    """(gm, its twin, xhat, scale) in g's dtype: da = W1^T g (fp32 W1) through the forward's ReLU mask, and the normalized y"""
    dt = g.dtype
    u = fw["used"]
    y, pre, s, mean, var = (u[k] for k in ("y", "pre", "s", "mean", "var"))
    n, c = g.shape[1], y.shape[1]
    W = _w1(w1, dt, defect == "da_packed_w1", defect).view(n, c, 1, 1)
    src = fw["value"]["out"] if defect == "da_wrong_operand" else g
    da, mda = _mm(W.transpose(0, 1), src), _mm(W.abs().transpose(0, 1), src.abs())
    keep = (pre < 0) if defect == "mask_side" else ((pre > 0) | torch.isnan(pre))
    gm, mg = torch.where(keep, da, torch.zeros_like(da)), torch.where(keep, mda, torch.zeros_like(mda))
    inv = _ch(1.0 / torch.sqrt(var.to(dt) + eps))
    return gm, mg, (y - _ch(mean.to(dt))) * inv, _ch(s.to(dt))


def _gammas(n, maps, h, w):
    """gamma along each gradient's longest path: the norm's backward, the pieces' sums and their fp64 sum, da's fmaf chain"""
    bnb = (BN_SUM + 8) * SUM + ELEM                                  # the norm's backward
    pieces = (maps * (-(-(h * w) // 4096)) + BN_SUM + 8) * SUM       # a piece sum, then the pieces' fp64 sum
    gda = (n + 1) * SUM                                              # da's fmaf chain
    return {"gy": gda + bnb, "gbw": gda + pieces + ELEM, "gbb": gda + pieces, "gW": pieces + ELEM, "gb": pieces}


def adjoint(fw, w1, b1, norm, g, training, eps, defect=None, totals=None, maps_total=None):
    """The adjoint of ``forward`` (as it used the run's statistics, when given) in g's dtype: da = W1^T g (fp32 W1), the norm's backward on
    (y, da) with the ReLU mask of the forward's fmaf, dW1 = g a^T, db1 = sum g; each with its absolute-value twin.  totals (optional):
    ``batch_totals`` of the whole batch when fw and g are a slice of it, whose per-channel sums the training dy then uses; maps_total: the
    whole batch's maps, for the reduction depths.  Returns (grads, bounds) keyed as GRAD_KEYS."""
    dt = g.dtype
    a = fw["used"]["a"]
    maps, c, h, w = a.shape
    n = g.shape[1]
    gm, mg, xhat, sc = _masked_da(fw, w1, g, eps, defect)
    if totals is None:
        cnt = maps * h * w
        t = {"s1": gm.sum((0, 2, 3)), "s2": (gm * xhat).sum((0, 2, 3)), "t1": mg.sum((0, 2, 3)), "t2": (mg * xhat.abs()).sum((0, 2, 3))}
    else:
        cnt, t = totals["count"], totals
    mean_of = lambda k: _ch(t[k]) / cnt                              # noqa: E731
    if training:
        dy = sc * (gm - mean_of("s1") - xhat * mean_of("s2"))
        mdy = sc.abs() * (mg + mean_of("t1") + xhat.abs() * mean_of("t2"))
    else:
        dy, mdy = sc * gm, sc.abs() * mg
    aw = gc.tf32_rz(a) if defect == "dw1_rz_a" else a
    gb = g.sum((0, 2, 3))
    grads = {"gy": dy, "gbw": (gm * xhat).sum((0, 2, 3)), "gbb": gm.sum((0, 2, 3)), "gW": _mm_w(aw, g).view(n, c),
             "gb": torch.zeros(n, dtype=dt, device=g.device) if defect == "bias_grad_dropped" else
             gb * c if defect == "db1_all_channels" else gb}
    twins = {"gy": mdy, "gbw": (mg * xhat.abs()).sum((0, 2, 3)), "gbb": mg.sum((0, 2, 3)), "gW": _mm_w(a.abs(), g.abs()).view(n, c),
             "gb": g.abs().sum((0, 2, 3))}
    gam = _gammas(n, maps_total or maps, h, w)
    for k, p in (("gbw", norm[0]), ("gbb", norm[1])):
        if p is None:
            grads[k] = twins[k] = None
    bounds = {k: (gam[k] * twins[k] if twins[k] is not None else None) for k in grads}
    return grads, bounds


def batch_totals(y, g, w1, b1, norm, mean, var, training, eps, chunk=1):
    """The whole batch's adjoint sums formed ``chunk`` maps at a time in fp64 (for a batch too large to restate at once): the per-channel
    sums of the masked da and da x^ with their twins ({"count", "s1", "s2", "t1", "t2"}, for ``adjoint``'s totals), and the parameter
    gradients dgamma, dbeta, dW1, db1 with their bounds (the sums of the per-map adjoints)"""
    maps, c, h, w = y.shape
    nd = [t.double() if t is not None else None for t in norm]
    t = {"count": maps * h * w}
    grads, bounds = {}, {}
    for j in range(0, maps, chunk):
        fw = forward(y[j:j + chunk].double(), w1, b1, nd, training, eps, True, (mean.double(), var.double()))
        gm, mg, xhat, _ = _masked_da(fw, w1, g[j:j + chunk].double(), eps)
        part = {"s1": gm.sum((0, 2, 3)), "s2": (gm * xhat).sum((0, 2, 3)), "t1": mg.sum((0, 2, 3)), "t2": (mg * xhat.abs()).sum((0, 2, 3))}
        gj, bj = adjoint(fw, w1, b1, nd, g[j:j + chunk].double(), False, eps, maps_total=maps)    # the sums need no batch terms
        for k, v in part.items():
            t[k] = t.get(k, 0) + v
        for k in ("gbw", "gbb", "gW", "gb"):
            if gj[k] is not None:
                grads[k], bounds[k] = grads.get(k, 0) + gj[k], bounds.get(k, 0) + bj[k]
    return t, grads, bounds


def stage_ratios(run, y, w1, b1, norm, training, eps, dtype=torch.float64):
    """{out / mean / var: (largest err / bound, non-finite elements agree)} of a run's [out, mean, var] against the fp64 restatement
    fed the run's statistics, and that restatement"""
    out, mean, var = (t.to(dtype) for t in run)
    nd = [t.to(dtype) if t is not None else None for t in norm]
    fw = forward(y.to(dtype), w1, b1, nd, training, eps, True, (mean, var))
    got = {"out": out, "mean": mean, "var": var}
    return {k: gc.excess(got[k], fw["value"][k], fw["bound"][k]) for k in got}, fw


def grad_ratios(fw, grads, w1, b1, norm, g, training, eps, dtype=torch.float64):
    """{gradient: (largest err / bound, non-finite agree)} of ``grads`` (GRAD_KEYS order, None where not computed) against the adjoint"""
    nd = [t.to(dtype) if t is not None else None for t in norm]
    want, bound = adjoint(fw, w1, b1, nd, g.to(dtype), training, eps)
    return {k: gc.excess(got.reshape(want[k].shape), want[k], bound[k]) for k, got in zip(GRAD_KEYS, grads)
            if got is not None and want[k] is not None}


# ------------------------------------------------------------------------------------------------------------------------------
# the module's running statistics
# ------------------------------------------------------------------------------------------------------------------------------
def running_update(rm, rv, mean, var, count, momentum, tracked, defect=None):
    """torch's BatchNorm update of (running_mean, running_var) from a batch's mean and biased var over ``count`` values per channel:
    factor = momentum (1 / num_batches_tracked after the increment when None), the variance moved toward the unbiased
    count / (count - 1) var.  defect "running_var_biased": toward the biased one.  In fp64, with a bound for fp32 bookkeeping."""
    f = 1.0 / tracked if momentum is None else momentum
    rm, rv, mean, var = (t.double() for t in (rm, rv, mean, var))
    v = var if defect == "running_var_biased" else var * (count / (count - 1))
    want_m, want_v = rm * (1 - f) + mean * f, rv * (1 - f) + v * f
    bound = lambda a, b, r: 8 * SUM * ((1 - f) * a.abs() + f * b.abs() + r.abs())        # noqa: E731
    return (want_m, bound(rm, mean, want_m)), (want_v, bound(rv, v, want_v))
