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
}


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
    if rounding:
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
    az = Z(a)
    out = _mm(W.view(*W.shape, 1, 1), az) + _ch(b1.to(dt))
    c = y.shape[1]
    bnd["out"] = (c + 3) * SUM * (_mm(W.abs().view(*W.shape, 1, 1), az.abs()) + _ch(b1.to(dt).abs())) + \
        _mm(W.abs().view(*W.shape, 1, 1), (Z(a_u) - az).abs())
    val["out"] = out
    used = {"y": y, "a": a, "pre": pre, "s": s, "mean": mean, "var": var}
    return {"value": val, "bound": bnd, "used": used, "rounding": rounding}


def adjoint(fw, w1, b1, norm, g, training, eps, defect=None):
    """The adjoint of ``forward`` (as it used the run's statistics, when given) in g's dtype: da = W1^T g (fp32 W1), the norm's backward on
    (y, da) with the ReLU mask of the forward's fmaf, dW1 = g a^T, db1 = sum g; each with its absolute-value twin.  Returns (grads,
    bounds) keyed as GRAD_KEYS."""
    dt = g.dtype
    u = fw["used"]
    y, a, pre, s, mean, var = (u[k] for k in ("y", "a", "pre", "s", "mean", "var"))
    maps, c, h, w = y.shape
    n = g.shape[1]
    W = _w1(w1, dt, False, defect).view(n, c, 1, 1)
    src = fw["value"]["out"] if defect == "da_wrong_operand" else g
    da, mda = _mm(W.transpose(0, 1), src), _mm(W.abs().transpose(0, 1), src.abs())
    keep = (pre < 0) if defect == "mask_side" else ((pre > 0) | torch.isnan(pre))
    gm, mg = torch.where(keep, da, torch.zeros_like(da)), torch.where(keep, mda, torch.zeros_like(mda))
    inv = _ch(1.0 / torch.sqrt(var.to(dt) + eps))
    xhat = (y - _ch(mean.to(dt))) * inv
    sc = _ch(s.to(dt))
    if training:
        dy = sc * (gm - gm.mean((0, 2, 3), keepdim=True) - xhat * (gm * xhat).mean((0, 2, 3), keepdim=True))
        mdy = sc.abs() * (mg + mg.mean((0, 2, 3), keepdim=True) + xhat.abs() * (mg * xhat.abs()).mean((0, 2, 3), keepdim=True))
    else:
        dy, mdy = sc * gm, sc.abs() * mg
    grads = {"gy": dy, "gbw": (gm * xhat).sum((0, 2, 3)), "gbb": gm.sum((0, 2, 3)), "gW": _mm_w(a, g).view(n, c),
             "gb": torch.zeros(n, dtype=dt, device=g.device) if defect == "bias_grad_dropped" else g.sum((0, 2, 3))}
    twins = {"gy": mdy, "gbw": (mg * xhat.abs()).sum((0, 2, 3)), "gbb": mg.sum((0, 2, 3)), "gW": _mm_w(a.abs(), g.abs()).view(n, c),
             "gb": g.abs().sum((0, 2, 3))}
    bnb = (BN_SUM + 8) * SUM + ELEM                                  # the norm's backward
    pieces = (maps * (-(-(h * w) // 4096)) + BN_SUM + 8) * SUM       # a piece sum, then the pieces' fp64 sum
    gda = (n + 1) * SUM                                              # da's fmaf chain
    gam = {"gy": gda + bnb, "gbw": gda + pieces + ELEM, "gbb": gda + pieces, "gW": pieces + ELEM, "gb": pieces}
    for k, p in (("gbw", norm[0]), ("gbb", norm[1])):
        if p is None:
            grads[k] = twins[k] = None
    bounds = {k: (gam[k] * twins[k] if twins[k] is not None else None) for k in grads}
    return grads, bounds


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
