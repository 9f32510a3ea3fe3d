"""Cases and restatements shared by tests/test_spatial_gru_cases_cpu.py and tests/test_spatial_gru_envelope_gpu.py: the shapes that walk
the SpatialGRU's (csrc/spatial_gru.cu) accepted envelope, TF32 rounding in its three modes, and a stage-by-stage restatement of the
GRU's steps and of their adjoint, each stage with an element-wise error bound.  Plain torch on any device; the convolutions are
built from ``unfold`` and a matmul, so a NaN lands on exactly the pixels a direct convolution puts it on.

The formulas are the header's (include/fiery_b200.h, fiery_spatial_gru_*).  Per step, with h the previous state:
  z = conv(tf32(W_gates), tf32([x_t, h])) + b_gates + bias_init,  u, r = 1 / (1 + exp(-z))  (the two halves of z)
  q = (1 - r) h,  s = conv(tf32(W_state), tf32([x_t, q]))
  scale = gamma / sqrt(var + eps), shift = beta - mean scale (fp64, rounded once to fp32),  a = max(fmaf(scale, s, shift), 0)
  h' = (1 - u) h + u a
and the adjoint in the order csrc/spatial_gru.cu gives: dh' = grad_out + carry -> da = u dh', dG_u = dh' (a - h) u (1 - u),
carry = (1 - u) dh'; the BN + ReLU backward -> ds; the state convolution's input gradient -> [dx_t, dq], dG_r = -dq h r (1 - r),
carry += (1 - r) dq; the gates' input gradient from [dG_u, dG_r] -> added to [dx_t, carry].  The weight gradients read their
activations rounded to nearest and the output gradient truncated (the tensor core drops its low bits).

Bounds.  Every quantity carries an absolute-value twin M: the same computation on |W|, |inputs| and every minus turned into a plus.
A computed value then lies within gamma * M of the exact one, where gamma adds, along the longest path to it, 2^-11 for each operand
rounded to TF32 to nearest, 2^-10 for each truncated one, n 2^-23 for each n-term fp32 or wgmma sum, and a few 2^-24 for each
fp32 elementwise operation.  The forward stages take the kernel's own inputs to each stage (its previous output, its r, its q, its
s, its statistics), whose TF32 rounding the restatement then repeats exactly, so their bounds hold the summation only."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24                  # fp32 unit roundoff
SUM = 2.0 ** -23                # per term of an fp32 or wgmma sum
RNA = 2.0 ** -11                # an operand rounded to TF32 to nearest
RZ = 2.0 ** -10                 # an operand truncated to TF32
BN_SUM = 32                     # terms along the batch norm's blocked piece sums (4 chunks, 4 lanes, 5 butterfly, 8 warps, slack)
ELEM = 16 * U                   # a step's elementwise fp32 operations


# ------------------------------------------------------------------------------------------------------------------------------
# TF32 rounding of fp32 values (held in any float dtype): 10 mantissa bits
# ------------------------------------------------------------------------------------------------------------------------------
def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float32).contiguous().view(torch.int32)


def _back(bits: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    """the rounded bits as like's dtype; a NaN stays NaN (adding the rounding bias to a NaN with a full payload, such as the GPU's
    0x7fffffff, would carry into the sign bit and make it -0)"""
    r = bits.view(torch.float32).to(like.dtype)
    return torch.where(torch.isnan(like), like, r)


def tf32_rna(t: torch.Tensor) -> torch.Tensor:
    """to nearest, ties away from zero (cvt.rna.tf32.f32)"""
    return _back((_bits(t) + 0x1000) & ~0x1FFF, t)


def tf32_rz(t: torch.Tensor) -> torch.Tensor:
    """toward zero (the low 13 bits dropped)"""
    return _back(_bits(t) & ~0x1FFF, t)


def tf32_rne(t: torch.Tensor) -> torch.Tensor:
    """to nearest, ties to even"""
    b = _bits(t)
    return _back((b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF, t)


def f32_round(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float32).to(t.dtype)


# ------------------------------------------------------------------------------------------------------------------------------
# 3x3 convolutions (zero padding 1) from unfold: forward, input gradient and weight gradient over (n, C, X, Y) maps
# ------------------------------------------------------------------------------------------------------------------------------
def conv(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    n, _, h, wd = x.shape
    cols = F.unfold(x, 3, padding=1)                                            # (n, C * 9, X * Y)
    return (w.reshape(w.shape[0], -1) @ cols).view(n, w.shape[0], h, wd)


def conv_t(g: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """the input gradient of conv(., w) from g"""
    return conv(g, w.transpose(0, 1).flip(2, 3))


def conv_w(x: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """the weight gradient of conv(x, .) from g: (O, C, 3, 3)"""
    cols = F.unfold(x, 3, padding=1)
    gw = torch.einsum("nop,nkp->ok", g.flatten(2), cols)
    return gw.view(g.shape[1], x.shape[1], 3, 3)


def _sigmoid(z):
    return 1.0 / (1.0 + torch.exp(-z))


def _sigmoid_slope(z_abs_lo):
    """the largest sigmoid'(z) over |z| >= z_abs_lo"""
    e = torch.exp(-z_abs_lo)
    return e / (1.0 + e) ** 2


# ------------------------------------------------------------------------------------------------------------------------------
# the restatement
# ------------------------------------------------------------------------------------------------------------------------------
def wgrad_depth(b: int, T: int, X: int, Y: int) -> int:
    """terms along the weight gradient's longest sum path: 8-pixel wgmma groups over a chunk's 32-pixel tiles, then the chunks"""
    tiles = b * T * X * ((Y + 31) // 32)
    chunks = min(tiles, 128)
    return -(-tiles // chunks) * 4 * 4 + chunks + 8


def forward(x, h0, p, frames: int, training: bool, eps: float, bias_init: float, rounding: bool = True, kernel=None):
    """The GRU's forward, stage by stage, in x's dtype.  x (b, Tx, C_x, X, Y), h0 (b, C_h, X, Y); p: dict of w_gates (2 C_h, C_x + C_h,
    3, 3), b_gates (2 C_h), w_state, gamma, beta (None: affine=False), running_mean, running_var.  kernel (optional): the kernel's
    out, u, r, q, s (T, b, C_h, X, Y each), means and vars, fed to each stage in place of the restatement's own.  rounding False
    computes the module's exact math (no TF32, no fp32 scale / shift).

    Returns a dict of per-step lists: value[stage] and bound[stage] for z, u, r, q, s, mean, var, out; plus what the adjoint needs
    (h, a, pre, scale, shift, the stage values the step used)."""
    R = tf32_rna if rounding else (lambda t: t)
    r32 = f32_round if rounding else (lambda t: t)
    b, tx, cx, X, Y = x.shape
    ch = h0.shape[1]
    wg, ws = R(p["w_gates"]), R(p["w_state"])
    n_g, n_s = 9 * (cx + ch) + 2, 9 * (cx + ch)
    keys = ("h", "x", "z", "u", "r", "q", "s", "mean", "var", "scale", "shift", "pre", "a", "out")
    val = {k: [] for k in keys}
    bnd = {k: [] for k in ("u", "r", "q", "s", "mean", "var", "out")}
    used = {k: [] for k in ("u", "r", "q", "s", "mean", "var")}
    for t in range(frames):
        h = h0 if t == 0 else (kernel["out"][:, t - 1] if kernel is not None else val["out"][-1])
        xt = x[:, t if tx > 1 else 0]
        xin = R(torch.cat([xt, h], 1))
        z = conv(xin, wg) + p["b_gates"].view(1, -1, 1, 1) + bias_init
        mz = conv(xin.abs(), wg.abs()) + p["b_gates"].abs().view(1, -1, 1, 1) + abs(bias_init)
        ez = (n_g * SUM + 2 * U) * mz
        g = _sigmoid(z)
        eg = _sigmoid_slope((z.abs() - ez).clamp_min(0)) * ez + 8 * U * g
        u, r = g[:, :ch], g[:, ch:]
        u_k = kernel["u"][t] if kernel is not None else u
        r_k = kernel["r"][t] if kernel is not None else r
        q = (1 - r_k) * h
        q_k = kernel["q"][t] if kernel is not None else q
        sin = R(torch.cat([xt, q_k], 1))
        s = conv(sin, ws)
        es = n_s * SUM * conv(sin.abs(), ws.abs())
        s_k = kernel["s"][t] if kernel is not None else s
        if training:
            mean = s_k.mean((0, 2, 3))
            var = s_k.var((0, 2, 3), unbiased=False)
            emean = BN_SUM * SUM * s_k.abs().mean((0, 2, 3))
            evar = 2 * BN_SUM * SUM * var + 4 * emean * (s_k - mean.view(1, -1, 1, 1)).abs().mean((0, 2, 3)) + emean ** 2
        else:
            mean, var = p["running_mean"].to(x.dtype), p["running_var"].to(x.dtype)
            emean = evar = torch.zeros_like(mean)
        mean_k = kernel["means"][t] if kernel is not None else mean
        var_k = kernel["vars"][t] if kernel is not None else var
        gamma = p["gamma"] if p.get("gamma") is not None else torch.ones_like(mean_k)
        beta = p["beta"] if p.get("beta") is not None else torch.zeros_like(mean_k)
        sc64 = gamma.double() / torch.sqrt(var_k.double() + eps)
        scale = r32(sc64.to(x.dtype))
        shift = r32((beta.double() - mean_k.double() * sc64).to(x.dtype))
        pre = scale.view(1, -1, 1, 1) * s_k + shift.view(1, -1, 1, 1)
        a = torch.where(pre < 0, torch.zeros_like(pre), pre)
        out = (1 - u_k) * h + u_k * a
        eout = 4 * U * ((1 - u_k) * h.abs() + u_k * ((scale.view(1, -1, 1, 1) * s_k).abs() + shift.abs().view(1, -1, 1, 1)))
        for k, v in (("h", h), ("x", xt), ("z", z), ("u", u), ("r", r), ("q", q), ("s", s), ("mean", mean), ("var", var),
                     ("scale", scale), ("shift", shift), ("pre", pre), ("a", a), ("out", out)):
            val[k].append(v)
        for k, v in (("u", eg[:, :ch]), ("r", eg[:, ch:]), ("q", 3 * U * q.abs()), ("s", es), ("mean", emean), ("var", evar),
                     ("out", eout)):
            bnd[k].append(v)
        for k, v in (("u", u_k), ("r", r_k), ("q", q_k), ("s", s_k), ("mean", mean_k), ("var", var_k)):
            used[k].append(v)
    return {"value": val, "bound": bnd, "used": used, "cx": cx, "ch": ch, "rounding": rounding}


def adjoint(fw, x, h0, p, grad_out, training: bool, eps: float):
    """The adjoint of ``forward``'s steps (as they used the kernel's values, when given), in grad_out's dtype, with each gradient's
    absolute-value twin and bound.  Returns (grads, bounds): x, h0, w_gates, b_gates, w_state, gamma, beta (None where there is no
    affine parameter)."""
    v, used = fw["value"], fw["used"]
    cx, ch = fw["cx"], fw["ch"]
    rounding = fw["rounding"]
    R = tf32_rna if rounding else (lambda t: t)
    RZt = tf32_rz if rounding else (lambda t: t)
    wg, ws = R(p["w_gates"]), R(p["w_state"])
    b, tx, _, X, Y = x.shape
    T = len(v["out"])
    count = b * X * Y
    step = 2 * RNA + (27 * ch + BN_SUM + 4) * SUM + 2 * ELEM       # gamma added per step along the backward's longest path
    carry = torch.zeros_like(h0)
    mc = torch.zeros_like(h0)
    gx = torch.zeros_like(x)
    mgx = torch.zeros_like(x)
    gwg, mwg = torch.zeros_like(p["w_gates"]), torch.zeros_like(p["w_gates"])
    gws, mws = torch.zeros_like(p["w_state"]), torch.zeros_like(p["w_state"])
    gbg, mbg = torch.zeros(2 * ch, dtype=x.dtype, device=x.device), torch.zeros(2 * ch, dtype=x.dtype, device=x.device)
    dgam, mgam = torch.zeros(ch, dtype=x.dtype, device=x.device), torch.zeros(ch, dtype=x.dtype, device=x.device)
    dbet, mbet = torch.zeros_like(dgam), torch.zeros_like(dgam)
    for t in reversed(range(T)):
        h, xt, a, pre = v["h"][t], v["x"][t], v["a"][t], v["pre"][t]
        u, r, q, s = used["u"][t], used["r"][t], used["q"][t], used["s"][t]
        mean, var = used["mean"][t], used["var"][t]
        scale = v["scale"][t].view(1, -1, 1, 1)
        dh = grad_out[:, t] + carry
        mdh = grad_out[:, t].abs() + mc
        da, mda = u * dh, u * mdh
        dgu = dh * (a - h) * (u * (1 - u))
        mgu = mdh * (a.abs() + h.abs()) * (u * (1 - u))
        carry, mc = (1 - u) * dh, (1 - u) * mdh
        keep = (pre > 0) | torch.isnan(pre)
        dy = torch.where(keep, da, torch.zeros_like(da))
        mdy = torch.where(keep, mda, torch.zeros_like(mda))
        inv = 1.0 / torch.sqrt(var + eps)
        xhat = (s - mean.view(1, -1, 1, 1)) * inv.view(1, -1, 1, 1)
        if training:
            m1, m2 = dy.mean((0, 2, 3), keepdim=True), (dy * xhat).mean((0, 2, 3), keepdim=True)
            ds = scale * (dy - m1 - xhat * m2)
            mds = scale.abs() * (mdy + mdy.mean((0, 2, 3), keepdim=True) + xhat.abs() * (mdy * xhat.abs()).mean((0, 2, 3), keepdim=True))
        else:
            ds, mds = scale * dy, scale.abs() * mdy
        dgam += (dy * xhat).sum((0, 2, 3))
        mgam += (mdy * xhat.abs()).sum((0, 2, 3))
        dbet += dy.sum((0, 2, 3))
        mbet += mdy.sum((0, 2, 3))
        sg, msg = conv_t(ds, ws), conv_t(mds, ws.abs())
        dq, mdq = sg[:, cx:], msg[:, cx:]
        dgr = -dq * h * (r * (1 - r))
        mgr = mdq * h.abs() * (r * (1 - r))
        carry, mc = carry + (1 - r) * dq, mc + (1 - r) * mdq
        dg, mdg = torch.cat([dgu, dgr], 1), torch.cat([mgu, mgr], 1)
        gg, mgg = conv_t(dg, wg), conv_t(mdg, wg.abs())
        carry, mc = carry + gg[:, cx:], mc + mgg[:, cx:]
        ti = t if tx > 1 else 0
        gx[:, ti] += sg[:, :cx] + gg[:, :cx]
        mgx[:, ti] += msg[:, :cx] + mgg[:, :cx]
        xin, sin = R(torch.cat([xt, h], 1)), R(torch.cat([xt, q], 1))
        gwg += conv_w(xin, RZt(dg))
        mwg += conv_w(xin.abs(), mdg.abs())
        gws += conv_w(sin, RZt(ds))
        mws += conv_w(sin.abs(), mds)
        gbg += dg.sum((0, 2, 3))
        mbg += mdg.sum((0, 2, 3))
    gam = T * step
    wd = wgrad_depth(b, T, X, Y) * SUM + RZ
    bsum = (T * b * (-(-X * Y // 256)) + 8) * SUM
    grads = {"x": gx, "h0": carry, "w_gates": gwg, "b_gates": gbg, "w_state": gws,
             "gamma": dgam if p.get("gamma") is not None else None, "beta": dbet if p.get("beta") is not None else None}
    bounds = {"x": gam * mgx, "h0": gam * mc, "w_gates": (gam + wd) * mwg, "b_gates": (gam + bsum) * mbg,
              "w_state": (gam + wd) * mws, "gamma": (gam + (T + BN_SUM) * SUM) * mgam, "beta": (gam + (T + BN_SUM) * SUM) * mbet}
    return grads, bounds


# ------------------------------------------------------------------------------------------------------------------------------
# comparison
# ------------------------------------------------------------------------------------------------------------------------------
def excess(got: torch.Tensor, want: torch.Tensor, bound: torch.Tensor):
    """(largest |got - want| / bound over the finite elements, whether the non-finite elements agree): NaN where want is NaN, the
    same infinity where want is infinite"""
    got, want, bound = got.double(), want.double(), bound.double()
    fin = torch.isfinite(want)
    same = bool(torch.equal(torch.isnan(got), torch.isnan(want)) and torch.equal(got[torch.isinf(want)], want[torch.isinf(want)])
                and bool(torch.isfinite(got[fin]).all()))
    if not bool(fin.any()):
        return 0.0, same
    err = (got[fin] - want[fin]).abs()
    ratio = err / bound[fin].clamp_min(1e-300)
    ratio = torch.where(err == 0, torch.zeros_like(ratio), ratio)
    return float(ratio.max()), same


# ------------------------------------------------------------------------------------------------------------------------------
# the shape list
# ------------------------------------------------------------------------------------------------------------------------------
# (cx, ch, X, Y, b, T, Tx, bias_init).  Every channel count below takes each side at least once, so N = round8(2 C_h) reaches every
# instantiation up to 128 and C_h in 33..60 a second weight-gradient block narrower than 64; X and Y run over single-tile, exact-tile,
# one-past and ragged 200 edges of the 8 x 16 tiles.
CHANNELS = (1, 7, 8, 9, 31, 32, 33, 48, 60, 63, 64)
_XS = (1, 7, 8, 9, 200)
_YS = (4, 12, 16, 20, 200)

# the existing whole-GRU cases (tests/test_spatial_gru_gpu.py CASES), as (cx, ch, X, Y, b, T, Tx, bias_init)
BASE_CASES = [
    (32, 64, 12, 16, 2, 4, 1, 0.0),
    (64, 64, 7, 12, 1, 5, 5, 0.0),
    (1, 8, 1, 4, 3, 1, 1, 0.0),
    (35, 29, 9, 20, 2, 4, 4, 0.0),
    (64, 1, 10, 8, 1, 4, 4, 0.0),
    (32, 64, 40, 24, 3, 4, 4, 0.0),
    (32, 48, 12, 16, 2, 4, 1, 0.0),
    (64, 40, 9, 20, 2, 5, 5, 0.0),
    (16, 24, 8, 12, 2, 3, 3, 0.75),
]


def _envelope():
    cases = []
    n = len(CHANNELS)
    for i, cx in enumerate(CHANNELS):
        ch = CHANNELS[(3 * i + 5) % n]
        for k in range(2):
            j = 2 * i + k
            X, Y = _XS[j % 5], _YS[(j + k + i) % 5]
            if X == 200 and Y == 200:
                Y = 20
            b = (1, 3)[j % 2]
            T = (1, 2, 5)[j % 3]
            Tx = T if (i + k) % 2 else 1
            bias_init = (0.0, 0.75, -0.5)[j % 3]
            cases.append((cx if k == 0 else ch, ch if k == 0 else cx, X, Y, b, T, Tx, bias_init))
    # the gates' widths N = 32, 40 and 56 the channel list above does not reach
    cases += [(16, 16, 8, 12, 2, 2, 2, 0.0), (20, 20, 9, 16, 1, 3, 1, 0.5), (28, 28, 7, 20, 3, 2, 2, -0.5)]
    # the full grid at the project's widths, with ragged tiles on both edges
    cases += [(32, 64, 200, 200, 1, 2, 2, 0.0), (64, 48, 200, 200, 3, 1, 1, 0.25)]
    return cases


CASES = BASE_CASES + _envelope()


def case_id(c) -> str:
    cx, ch, X, Y, b, T, Tx, g = c
    return f"cx{cx}_ch{ch}_{X}x{Y}_b{b}_T{T}_Tx{Tx}" + (f"_g{g}" if g else "")


def params(cx: int, ch: int, seed: int, dtype=torch.float64, device="cpu", affine: bool = True):
    """random parameters at the scale of a trained GRU: weights ~ 1/sqrt(fan-in), biases, gamma near 1, running statistics"""
    g = torch.Generator().manual_seed(seed)
    fan = 9 * (cx + ch)
    p = {
        "w_gates": torch.randn(2 * ch, cx + ch, 3, 3, generator=g) * (1.5 / math.sqrt(fan)),
        "b_gates": torch.randn(2 * ch, generator=g) * 0.5,
        "w_state": torch.randn(ch, cx + ch, 3, 3, generator=g) * (1.5 / math.sqrt(fan)),
        "gamma": 1 + 0.3 * torch.randn(ch, generator=g) if affine else None,
        "beta": 0.3 * torch.randn(ch, generator=g) if affine else None,
        "running_mean": 0.1 * torch.randn(ch, generator=g),
        "running_var": torch.rand(ch, generator=g) + 0.5,
    }
    # every parameter an fp32 value, so the fp32 kernels and the fp64 restatement hold the same numbers
    return {k: (v.float().to(dtype=dtype, device=device) if v is not None else None) for k, v in p.items()}


def inputs(b, T, Tx, cx, ch, X, Y, seed, dtype=torch.float64, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, Tx, cx, X, Y, generator=g)
    h0 = torch.randn(b, ch, X, Y, generator=g)
    go = torch.randn(b, T, ch, X, Y, generator=g)
    return tuple(t.to(dtype=dtype, device=device) for t in (x, h0, go))


# ------------------------------------------------------------------------------------------------------------------------------
# checks of a run (the kernels', or an fp32 restatement's) against the fp64 restatement fed that run's own stage inputs
# ------------------------------------------------------------------------------------------------------------------------------
def as_kernel(out, saved, means, vars_):
    """the dict ``forward(kernel=...)`` takes, from a run's out (b, T, C_h, X, Y), saved (u, r, q, s stacked on a leading axis of 4, or
    flat), means and vars (T, C_h)"""
    b, T, ch, X, Y = out.shape
    s4 = saved.reshape(4, T, b, ch, X, Y)
    return {"out": out, "u": s4[0], "r": s4[1], "q": s4[2], "s": s4[3], "means": means, "vars": vars_}


def stage_ratios(run, x, h0, p, frames, training, eps, bias_init, dtype=torch.float64):
    """{stage: (largest err / bound over the steps, non-finite elements agree)} for u, r, q, s, mean, var, out, and the fp64
    restatement fed ``run`` (an ``as_kernel`` dict)"""
    k = {n: t.to(dtype) for n, t in run.items()}
    pd = {n: (t.to(dtype) if t is not None else None) for n, t in p.items()}
    fw = forward(x.to(dtype), h0.to(dtype), pd, frames, training, eps, bias_init, True, k)
    got = {"u": k["u"], "r": k["r"], "q": k["q"], "s": k["s"], "mean": k["means"], "var": k["vars"],
           "out": k["out"].transpose(0, 1)}
    res = {}
    for st, g in got.items():
        ratio, same = 0.0, True
        for t in range(frames):
            rr, ss = excess(g[t], fw["value"][st][t], fw["bound"][st][t])
            ratio, same = max(ratio, rr), same and ss
        res[st] = (ratio, same)
    return res, fw


def grad_ratios(fw, grads, x, h0, p, grad_out, training, eps, dtype=torch.float64):
    """{gradient: (largest err / bound, non-finite elements agree)} of ``grads`` (x, h0, w_gates, b_gates, w_state, gamma, beta)
    against the fp64 adjoint of ``fw`` (``stage_ratios``' restatement, which used the run's saved values)"""
    pd = {n: (t.to(dtype) if t is not None else None) for n, t in p.items()}
    want, bound = adjoint(fw, x.to(dtype), h0.to(dtype), pd, grad_out.to(dtype), training, eps)
    return {n: excess(grads[n], want[n], bound[n]) for n in want if want[n] is not None and grads.get(n) is not None}


# ------------------------------------------------------------------------------------------------------------------------------
# whole-module yardstick: fp64 with every convolution's operands rounded to TF32 (the kernels' operand rounding, not their order)
# ------------------------------------------------------------------------------------------------------------------------------
def _tf32_passthrough(t: torch.Tensor) -> torch.Tensor:
    """t rounded to TF32 (to nearest, ties away), the gradient passed straight through"""
    return t + (tf32_rna(t.detach()) - t).detach()


def tf32_operands(m: torch.nn.Module) -> torch.nn.Module:
    """m (an fp64 copy) with every Conv2d's input and weight rounded to TF32 first"""
    for c in m.modules():
        if isinstance(c, torch.nn.Conv2d):
            c.forward = (lambda c: lambda x: F.conv2d(_tf32_passthrough(x), _tf32_passthrough(c.weight), c.bias, c.stride,
                                                      c.padding))(c)
    return m


# ------------------------------------------------------------------------------------------------------------------------------
# the exact regime: eval, gates at exactly 0.5, eps 0, running_var 4, dyadic values, so that every TF32 operand is exact and every
# fp32 sum is exact; then any summation order gives the same bits
# ------------------------------------------------------------------------------------------------------------------------------
GRAIN = 2.0 ** -20              # every value a multiple of this
EXACT_LIMIT = 2.0 ** 4          # every value below this: 2^24 grains, so each fp32 value on the grain is exact


def exact_case(config: int, b=2, T=1, cx=4, ch=8, X=9, Y=20, seed=0):
    """(x, h0, p, grad_out) in fp64.  config 0: zero gate weights and biases; config 1: x = 0 and nonzero x-weights in the gates
    (the h-weights zero), so the gates are still 0.5 and their input gradient reaches dx."""
    g = torch.Generator().manual_seed(seed)
    q = lambda shape, lo, hi, step: torch.randint(lo, hi + 1, shape, generator=g).double() * step   # noqa: E731
    x = q((b, T, cx, X, Y), -2, 2, 0.25) if config == 0 else torch.zeros(b, T, cx, X, Y, dtype=torch.float64)
    h0 = q((b, ch, X, Y), -2, 2, 0.25)
    wg = torch.zeros(2 * ch, cx + ch, 3, 3, dtype=torch.float64)
    if config == 1:
        wg[:, :cx] = q((2 * ch, cx, 3, 3), -1, 1, 0.125)
    p = {"w_gates": wg, "b_gates": torch.zeros(2 * ch, dtype=torch.float64),
         "w_state": q((ch, cx + ch, 3, 3), -1, 1, 0.125) * (q((ch, cx + ch, 3, 3), 0, 1, 1.0)),
         "gamma": q((ch,), 2, 4, 0.5), "beta": q((ch,), -2, 2, 0.25),
         "running_mean": q((ch,), -2, 2, 0.125), "running_var": torch.full((ch,), 4.0, dtype=torch.float64)}
    go = q((b, T, ch, X, Y), -1, 1, 0.25)
    return x, h0, p, go


def _on_grain(t):
    v = t[torch.isfinite(t)] / GRAIN
    return bool(torch.equal(v, v.round()))


def exact_regime_holds(fw, grads, x, h0, p, go) -> list:
    """what breaks exactness in the restatement (empty: every convolution operand is TF32-exact and on the grain, every value and
    every absolute-value sum below EXACT_LIMIT, the gates exactly 0.5): the names of the offending quantities"""
    bad = []
    v = fw["value"]
    ops = {"w_gates": p["w_gates"], "w_state": p["w_state"]}
    for t in range(len(v["out"])):
        ops.update({f"xin{t}": torch.cat([v["x"][t], v["h"][t]], 1), f"sin{t}": torch.cat([v["x"][t], v["q"][t]], 1),
                    f"u{t}": v["u"][t], f"r{t}": v["r"][t], f"s{t}": v["s"][t], f"out{t}": v["out"][t]})
    ops.update({f"d_{k}": g for k, g in grads.items() if g is not None})
    for k, t in ops.items():
        if not (torch.equal(tf32_rna(t), t) or not (k.startswith(("xin", "sin", "w_")))) or not _on_grain(t) or t.abs().max() >= EXACT_LIMIT:
            bad.append(k)
    for t in range(len(v["out"])):
        if not (bool((v["u"][t] == 0.5).all()) and bool((v["r"][t] == 0.5).all())):
            bad.append(f"gates{t}")
    return bad
