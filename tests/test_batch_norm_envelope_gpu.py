"""GPU: the fused BatchNorm3d (csrc/batch_norm.cu) across the range its C ABI accepts, with the cases and restatements of
tests/_batch_norm_cases.py.

A  exact cases (every intermediate exact) bit for bit against the header's formulas: every mode on a few shapes and every shape of
   the list in one mode, through the C ABI from NaN-poisoned inputs into sentinel-guarded outputs and a workspace of exactly its
   size; eps 0 and a power-of-two eps, the latter also against fp64 F.batch_norm;
B  random data against the pieces' order model and the header's arithmetic: the mean's bits, dβ's bits, y = fmaf(scale, x, shift),
   the ReLU mask from the kernel's own output, eval's dx = scale * g';
C  hard statistics (|μ|/σ up to 1e5, σ far below √eps, constant channels, γ < 0 and 0, eps up to 0.1, magnitudes 1e±15) against
   fp64, within 3x torch's fp32 CUDA error;
D  NaN and ±inf against torch: eval pixel by pixel in every mode, one NaN channel in training;
E  layouts and host routes bit-identical to the contiguous call: stride-0 expansions, channel slices, frame-major views, 4-byte
   misalignment of every pointer the kernels branch on, fp16 / bf16, an expanded grad_y, a strided residual, every backward subset;
F  FusedBatchNorm3d over several training steps of different shapes and then eval, against an fp64 nn.BatchNorm3d;
G  one whole swapped TemporalModel at the shipped 200 x 200 grid against the fp64 oracle."""
import copy
import itertools

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from fiery_b200 import _lib, ops  # noqa: F401  (registers the operators)
from fiery_b200.batch_norm import FusedBatchNorm3d
from fiery_b200.batch_norm import backward as bn_backward
from fiery_b200.batch_norm import forward as bn_forward
from oracle import temporal_oracle as TO
from tests import _batch_norm_cases as BC
from tests import _temporal_cases as TC
from tests.test_batch_norm_gpu import _model, _no_tf32, _step, _swapped  # noqa: F401  (_no_tf32: the module's fixture)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
_ids = lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v)     # noqa: E731


def _nerr(a, b):
    return TO.normwise_error(a, b)


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _np(t):
    return t.detach().cpu().numpy()


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


# ------------------------------------------------------------------------------------------------------------------------------
# the C ABI on guarded buffers
# ------------------------------------------------------------------------------------------------------------------------------
def _desc(x, training, relu, eps):
    b, c, s = x.shape[:3]
    d = _lib.BatchNormDesc()
    d.batch, d.channels, d.frames, d.pixels = b, c, s, int(np.prod(x.shape[3:]))
    d.stride_b, d.stride_c, d.stride_t = x.stride(0), x.stride(1), x.stride(2)
    d.training, d.relu, d.eps = int(training), int(relu), float(eps)
    return d


def _ptr(t):
    return 0 if t is None else t.data_ptr()


class _Workspace:
    """exactly fiery_batch_norm_workspace_bytes(d) bytes, NaN-filled, between sentinel margins"""

    def __init__(self, d):
        nbytes = int(_lib.load().fiery_batch_norm_workspace_bytes(d))
        assert nbytes > 0 and nbytes % 8 == 0
        self.buf, self.view = TC.guarded(nbytes // 4, 256, 256, DEV)

    def check(self):
        TC.assert_written_and_contained(self.buf, self.view, "workspace", must_write=False)


def abi_forward(x, w, b, rm, rv, r, training, relu, eps):
    """fiery_batch_norm_forward into guarded outputs: (y (b, C, s, pixels), mean, var), every store checked to stay inside"""
    d = _desc(x, training, relu, eps)
    bsz, c, s = x.shape[:3]
    n = bsz * c * s * d.pixels
    ws = _Workspace(d)
    yb, y = TC.guarded(n, 64, 64, DEV)
    mb, mean = TC.guarded(c, 64, 64, DEV)
    vb, var = TC.guarded(c, 64, 64, DEV)
    _lib.call("fiery_batch_norm_forward", DEV, d, x.data_ptr(), _ptr(w), _ptr(b), _ptr(rm), _ptr(rv), _ptr(r), y.data_ptr(),
              mean.data_ptr(), var.data_ptr(), ws.view.data_ptr())
    torch.cuda.synchronize()
    for buf, view, what in ((yb, y, "y"), (mb, mean, "mean"), (vb, var, "var")):
        TC.assert_written_and_contained(buf, view, what, must_write=False)
    ws.check()
    return y.view(bsz, c, s, d.pixels), mean, var


def abi_backward(x, dy, w, b, mean, var, training, relu, eps, need=(True, True, True)):
    """fiery_batch_norm_backward into guarded outputs, NULL where `need` says no (their guarded buffers must stay untouched):
    (dx, dw, db), None where not asked for"""
    d = _desc(x, training, relu, eps)
    bsz, c, s = x.shape[:3]
    n = bsz * c * s * d.pixels
    ws = _Workspace(d)
    outs = [TC.guarded(n, 64, 64, DEV), TC.guarded(c, 64, 64, DEV), TC.guarded(c, 64, 64, DEV)]
    ptrs = [view.data_ptr() if k else 0 for k, (_, view) in zip(need, outs)]
    _lib.call("fiery_batch_norm_backward", DEV, d, x.data_ptr(), dy.data_ptr(), _ptr(w), _ptr(b), mean.data_ptr(), var.data_ptr(),
              *ptrs, ws.view.data_ptr())
    torch.cuda.synchronize()
    for k, (buf, view), what in zip(need, outs, ("dx", "dweight", "dbias")):
        if k:
            TC.assert_written_and_contained(buf, view, what, must_write=False)
        else:                                                   # a NULL output: its buffer is as it was
            assert bool(view.isnan().all()) and bool((buf[:64] == TC.SENTINEL).all()) and bool((buf[-64:] == TC.SENTINEL).all()), what
    ws.check()
    got = [view if k else None for k, (_, view) in zip(need, outs)]
    if got[0] is not None:
        got[0] = got[0].view(bsz, c, s, d.pixels)
    return tuple(got)


def _written(*ts):
    """no output element was left NaN (the exact and random cases have finite results)"""
    for t in ts:
        if t is not None:
            assert not bool(t.isnan().any())


# ------------------------------------------------------------------------------------------------------------------------------
# A: exact cases, bit for bit
# ------------------------------------------------------------------------------------------------------------------------------
def _run_exact(case, shape, training, relu, residual, affine):
    x = TC.poisoned(torch.from_numpy(case["x"]), DEV)
    w, b = (_t(case["w"]), _t(case["b"])) if affine else (None, None)
    rm, rv = _t(case["rm"]), _t(case["rv"])
    r = TC.poisoned(torch.from_numpy(case["r"]), DEV) if residual else None
    dy = TC.poisoned(torch.from_numpy(case["dy"]), DEV)
    eps = case["eps"]
    y, mean, var = abi_forward(x, w, b, None if training else rm, None if training else rv, r, training, relu, eps)
    dx, dw, db = abi_backward(x, dy, w, b, mean, var, training, relu, eps)
    _written(y, mean, var, dx, dw, db)
    want = BC.restate(case["x"], case["w"] if affine else None, case["b"] if affine else None, case["rm"], case["rv"],
                      case["r"] if residual else None, case["dy"], training, relu, eps)
    for name, got in (("mean", mean), ("var", var), ("y", y), ("dx", dx), ("dw", dw), ("db", db)):
        assert _bits_equal(_np(got), want[name]), f"{shape} {name}: {np.abs(_np(got).astype(np.float64) - want[name]).max():.3e}"
    return x, w, b, rm, rv, r, dy, (y, mean, var, dx, dw, db)


MODES = list(itertools.product([True, False], [True, False], [True, False], [True, False]))   # training, relu, residual, affine
MODE_SHAPES = [(2, 3, 1, 1, 4097), (1, 129, 1, 1, 2), (2, 4, 3, 200, 200)]


@pytest.mark.parametrize("shape", MODE_SHAPES, ids=_ids)
def test_exact_every_mode(shape):
    for affine in (True, False):
        case = BC.exact_case(shape, seed=sum(shape), affine=affine)
        for training, relu, residual, _ in MODES[::2]:
            _run_exact(case, shape, training, relu, residual, affine)


@pytest.mark.parametrize("shape", BC.SHAPE_LIST, ids=_ids)
def test_exact_every_shape(shape):
    case = BC.exact_case(shape, seed=sum(shape) + 1)
    got = _run_exact(case, shape, True, True, True, True)[-1]
    # the ReLU's equality case was met: some pre-activations are exactly 0
    scale, shift = BC.scale_shift(case["w"], case["b"], _np(got[1]), _np(got[2]), case["eps"])[:2]
    pre = BC.fmaf_exact(scale.reshape(1, -1, 1, 1), case["x"], shift.reshape(1, -1, 1, 1))
    assert np.any(pre == 0)


@pytest.mark.parametrize("shape,eps", [((2, 3, 1, 1, 4097), 8.0), ((2, 129, 1, 1, 2), 8.0), ((2, 4, 3, 200, 200), 8.0),
                                       ((2, 3, 1, 1, 1), 1.0)], ids=_ids)
def test_exact_with_eps_against_fp64_batch_norm(shape, eps):
    case = BC.exact_case(shape, seed=7, eps=eps)
    for training, relu in itertools.product((True, False), (True, False)):
        x, w, b, rm, rv, r, dy, got = _run_exact(case, shape, training, relu, True, True)
        xd = x.double().reshape(*shape).requires_grad_(True)
        wd, bd = w.double().requires_grad_(True), b.double().requires_grad_(True)
        yd = F.batch_norm(xd, rm.double().clone(), rv.double().clone(), wd, bd, training, 0.1, eps)
        scale, shift = BC.scale_shift(case["w"], case["b"], _np(got[1]), _np(got[2]), eps)[:2]
        # |dy| <= 2^-24 (|scale x| + |shift|) + ulp(y) / 2: the rounding of the two fp32 coefficients, then of y
        pre = _np(yd.detach()).reshape(case["x"].shape)
        bar = 2.0 ** -24 * (np.abs(scale.reshape(1, -1, 1, 1) * case["x"]) + np.abs(shift.reshape(1, -1, 1, 1))) + \
            np.spacing(np.abs(pre).astype(np.float32)) / 2
        yk = _np(got[0]).astype(np.float64) - case["r"]
        ref = np.maximum(pre, 0) if relu else pre
        assert np.all(np.abs(yk - ref) <= bar), float(np.max(np.abs(yk - ref) - bar))


def test_exact_eps_zero_through_the_host():
    shape = (2, 3, 2, 1, 4097)
    case = BC.exact_case(shape, seed=3)
    x = _t(case["x"]).view(shape)
    for training in (True, False):
        y, mean, var = bn_forward(x, _t(case["w"]), _t(case["b"]), _t(case["rm"]), _t(case["rv"]), _t(case["r"]).view(shape), training,
                                  0.0, True)
        dx, dw, db = bn_backward(_t(case["dy"]).view(shape), x, _t(case["w"]), _t(case["b"]), mean, var, training, 0.0, True, True,
                                 True, True)
        want = BC.restate(case["x"], case["w"], case["b"], case["rm"], case["rv"], case["r"], case["dy"], training, True, 0.0)
        for name, got in (("mean", mean), ("var", var), ("y", y), ("dx", dx), ("dw", dw), ("db", db)):
            assert _bits_equal(_np(got).reshape(want[name].shape), want[name]), name


# ------------------------------------------------------------------------------------------------------------------------------
# B: random data against the order model
# ------------------------------------------------------------------------------------------------------------------------------
B_SHAPES = [(1, 3, 1, 64, 64), (1, 35, 1, 1, 4093), (1, 2, 1, 1, 7), (2, 4, 3, 200, 200), (1, 2, 1, 1, 8193), (4, 2, 5000, 1, 2),
            (3, 129, 2, 1, 4099)]


def _random(shape, seed):
    rng = np.random.default_rng(seed)
    b, c, s, X, Y = shape
    p = X * Y
    x = (rng.standard_normal((b, c, s, p)) * np.exp2(rng.integers(-3, 4, (b, c, s, p))) +
         rng.standard_normal(c).reshape(1, c, 1, 1) * 4).astype(np.float32)
    w = (rng.standard_normal(c) * 1.5).astype(np.float32)
    w[::5] = -np.abs(w[::5])
    bias = rng.standard_normal(c).astype(np.float32)
    rm = rng.standard_normal(c).astype(np.float32)
    rv = (rng.random(c) * 3 + 0.1).astype(np.float32)
    r = rng.standard_normal((b, c, s, p)).astype(np.float32)
    dy = rng.standard_normal((b, c, s, p)).astype(np.float32)
    return x, w, bias, rm, rv, r, dy


def _either(got, a, b_):
    """per channel (axis 1, or axis 0 of a (C,) vector), got's bits are a's or b_'s"""
    got, a, b_ = (np.asarray(t, np.float32) for t in (got, a, b_))
    ax = tuple(i for i in range(got.ndim) if i != (1 if got.ndim > 1 else 0))
    ok_a = np.all(got.view(np.int32) == a.view(np.int32), axis=ax) if ax else got.view(np.int32) == a.view(np.int32)
    ok_b = np.all(got.view(np.int32) == b_.view(np.int32), axis=ax) if ax else got.view(np.int32) == b_.view(np.int32)
    return np.all(ok_a | ok_b), np.flatnonzero(~(ok_a | ok_b))


@pytest.mark.parametrize("shape", B_SHAPES, ids=_ids)
def test_random_data_against_the_order_model(shape):
    x, w, bias, rm, rv, r, dy = _random(shape, seed=sum(shape))
    b, c, s, X, Y = shape
    p = X * Y
    xs, dys = TC.poisoned(torch.from_numpy(x), DEV), TC.poisoned(torch.from_numpy(dy), DEV)
    wt, bt, rmt, rvt = _t(w), _t(bias), _t(rm), _t(rv)
    counts = np.tile(BC.piece_counts(p), b * s)
    pm = BC.bn_piece_sums_model(x, p) / BC.piece_counts(p)
    if b * s * len(BC.piece_sizes(p)) == 1:
        merged = (pm[0, :, 0, 0], pm[0, :, 0, 0])
    else:
        m2 = np.zeros_like(pm)                                       # the mean does not depend on the pieces' M2
        merged = (BC.chan_merge(BC.channel_pieces(pm, p), BC.channel_pieces(m2, p), counts, False)[0],
                  BC.chan_merge(BC.channel_pieces(pm, p), BC.channel_pieces(m2, p), counts, True)[0])
    for training, relu, residual in [(True, True, False), (True, False, True), (False, True, False), (False, False, True)]:
        rt = TC.poisoned(torch.from_numpy(r), DEV) if residual else None
        y, mean, var = abi_forward(xs, wt, bt, None if training else rmt, None if training else rvt, rt, training, relu, 1e-5)
        dx, dw, db = abi_backward(xs, dys, wt, bt, mean, var, training, relu, 1e-5)
        _written(y, mean, var, dx, dw, db)
        mean_, var_, y_, dx_, db_ = _np(mean), _np(var), _np(y), _np(dx), _np(db)
        if training:
            ok, bad = _either(mean_, *merged)
            assert ok, f"mean of channels {bad[:8]}"
        else:
            assert _bits_equal(mean_, rm) and _bits_equal(var_, rv)
        # y = fmaf(scale, x, shift) (+ ReLU, + residual), scale and shift from the kernel's own statistics, either shift rounding
        scale, sh_u, sh_c = BC.scale_shift(w, bias, mean_, var_, 1e-5)
        ys = []
        for sh in (sh_u, sh_c):
            pre = BC.fmaf_exact(scale.reshape(1, -1, 1, 1), x, sh.reshape(1, -1, 1, 1))
            yy = np.where(pre < 0, np.float32(0), pre) if relu else pre
            ys.append((yy + r).astype(np.float32) if residual else yy)
        ok, bad = _either(y_, *ys)
        assert ok, f"y of channels {bad[:8]}"
        # dβ: the fp64 ascending sum of the pieces' fp32 sums of g', the mask the kernel's own y > 0 when y is the ReLU's output
        g = np.where(y_ > 0, dy, np.float32(0)) if relu else dy
        want_db = BC.seq_sum64(BC.channel_pieces(BC.bn_piece_sums_model(g, p), p)).astype(np.float32)
        assert _bits_equal(db_, want_db), f"dbias: {np.abs(db_ - want_db).max():.3e}"
        if not training:
            assert _bits_equal(dx_, (scale.reshape(1, -1, 1, 1) * g).astype(np.float32)), "eval dx = scale * g'"
            if relu:
                assert np.array_equal(dx_ != 0, y_ > 0), "eval dx is nonzero exactly where y > 0"
        if relu and not residual:
            _, _, db1 = abi_backward(xs, torch.ones_like(dys), wt, bt, mean, var, training, relu, 1e-5, (False, False, True))
            assert np.array_equal(_np(db1), (y_ > 0).sum((0, 2, 3)).astype(np.float32)), "dbias with dy = 1: the positive outputs"


def test_order_shows_in_the_mean():
    """2^24 and two 1.0s per piece (tests/test_batch_norm_cases_cpu.py: the model's order on chosen values): the means' bits tell
    (p0 + p1) + (p2 + p3) from a left-to-right chunk sum"""
    x = np.zeros((1, 4, 1, 4096), np.float32)
    for ch, at in enumerate(((0, 2, 3), (0, 1, 2), (1024, 0, 1), (0, 4, 68))):
        x[0, ch, 0, at[0]] = 2.0 ** 24
        x[0, ch, 0, at[1]] = x[0, ch, 0, at[2]] = 1.0
    xs = TC.poisoned(torch.from_numpy(x), DEV)
    _, mean, _ = abi_forward(xs, None, None, None, None, None, True, False, 1e-5)
    want = BC.bn_piece_sums_model(x, 4096)[0, :, 0, 0] / np.float32(4096)
    assert _bits_equal(_np(mean), want) and len(set(want.tolist())) == 2


# ------------------------------------------------------------------------------------------------------------------------------
# C: hard statistics against fp64
# ------------------------------------------------------------------------------------------------------------------------------
def _torch_stats(x, w, b, gy, eps, dtype):
    """F.batch_norm + ReLU in training, in dtype on the device: (y, biased var, dx, dw, db, mean); the statistics from the running
    ones with momentum 1 (torch's batch mean and unbiased batch variance, times (n - 1) / n)"""
    xi = x.detach().to(dtype).clone().requires_grad_(True)
    wi, bi = w.to(dtype).clone().requires_grad_(True), b.to(dtype).clone().requires_grad_(True)
    c = x.shape[1]
    rm, rv = torch.zeros(c, dtype=dtype, device=DEV), torch.ones(c, dtype=dtype, device=DEV)
    y = F.relu(F.batch_norm(xi, rm, rv, wi, bi, True, 1.0, eps))
    y.backward(gy.to(dtype))
    n = x.numel() // c
    return y.detach(), rv.double() * (n - 1) / n, xi.grad, wi.grad, bi.grad, rm.double()


def _hard_case(kind, eps):
    g = torch.Generator().manual_seed(("offsets", "flat", "magnitudes").index(kind) * 100 + round(-np.log10(eps)))
    shape = (2, 6, 3, 200, 200)
    z = torch.randn(shape, generator=g, dtype=torch.float64)
    w = torch.tensor([1.0, -1.5, 0.0, 0.75, 2.0, -0.25], dtype=torch.float64)
    b = torch.tensor([0.1, -0.2, 0.3, 0.0, -0.5, 0.25], dtype=torch.float64)
    if kind == "offsets":                                           # |mu| / sigma = 0, 1e2, 1e3, 1e4, 1e5, -1e4
        ratio = torch.tensor([0.0, 1e2, 1e3, 1e4, 1e5, -1e4], dtype=torch.float64)
        x = z * 0.5 + (ratio * 0.5).view(1, -1, 1, 1, 1)
    elif kind == "flat":                                            # sigma far below sqrt(eps), and constant channels (0, and 0.375
        sig = torch.tensor([1e-6, 1e-4, 0.0, 0.0, 1e-5, 3e-3], dtype=torch.float64) * eps ** 0.5   # under gamma = 0)
        # a constant whose piece sums round (0.1) has a mean a few ulps off, and then dweight = ulp(mu) * sum dy / sqrt(eps) where
        # torch's is 0; 0.375's sums are exact
        x = z * sig.view(1, -1, 1, 1, 1) + torch.tensor([0.0, 0.0, 0.375, 0.0, 0.0, 0.0], dtype=torch.float64).view(1, -1, 1, 1, 1)
        b[3] = 0.5                                                  # the constant 0 channel's output away from the ReLU's kink
    else:                                                           # magnitudes near 1e-15 and 1e15
        mag = torch.tensor([1e-15, 1e15, 1e-15, 1e15, 3e-15, 3e14], dtype=torch.float64)
        x = (z + torch.tensor([0.0, 0.0, 5.0, 5.0, 1.0, -2.0], dtype=torch.float64).view(1, -1, 1, 1, 1)) * mag.view(1, -1, 1, 1, 1)
    gy = torch.randn(shape, generator=g)
    return x.float().to(DEV), w.float().to(DEV), b.float().to(DEV), gy.to(DEV)


HARD = [("offsets", 1e-5), ("flat", 1e-5), ("flat", 1e-3), ("flat", 0.1), ("magnitudes", 1e-5), ("offsets", 0.1)]


@pytest.mark.parametrize("kind,eps", HARD, ids=str)
def test_hard_statistics_against_fp64(kind, eps):
    x, w, b, gy = _hard_case(kind, eps)
    y, mean, var = bn_forward(x, w, b, None, None, None, True, eps, True)
    dx, dw, db = bn_backward(gy, x, w, b, mean, var, True, eps, True, True, True, True)
    want = _torch_stats(x, w, b, gy, eps, torch.float64)
    theirs = _torch_stats(x, w, b, gy, eps, torch.float32)
    var64, mean64 = want[1], want[5]
    # the statistics channel by channel: within 3x torch's own error, or a few fp32 roundings of the exact value; a constant
    # channel's var is 0 up to the square of a few roundings of its mean
    err, err_t = (var.double() - var64).abs(), (theirs[1] - var64).abs()
    floor = torch.where(var64 == 0, (2.0 ** -22 * mean64.abs()) ** 2, 4 * 2.0 ** -24 * var64)
    assert bool((err <= torch.maximum(3 * err_t, floor)).all()), f"var: {err.tolist()} torch {err_t.tolist()} exact {var64.tolist()}"
    merr, merr_t = (mean.double() - mean64).abs(), (theirs[5] - mean64).abs()
    mfloor = 4 * 2.0 ** -24 * (mean64.abs() + var64.sqrt())
    assert bool((merr <= torch.maximum(3 * merr_t, mfloor)).all()), f"mean: {merr.tolist()} torch {merr_t.tolist()}"
    if kind == "offsets":                                           # and an absolute bar where |mu| / sigma <= 1e4
        rel = (err / var64).tolist()
        assert max(rel[i] for i in (0, 1, 2, 3, 5)) <= 1e-5, rel
    # the outputs: y = fmaf(scale, x, shift) with shift = beta - mean * scale rounded to fp32 carries |mean * scale| 2^-24, which at
    # |mu| / sigma = 1e5 is 6e-3 of the output's spread and moves the ReLU's mask (the header's arithmetic, bounded in A); there the
    # statistics above are checked, the outputs of the other channels here
    keep = [0, 1, 2, 3, 5] if kind == "offsets" else list(range(6))
    for name, a, t, e in (("y", y, theirs[0], want[0]), ("dx", dx, theirs[2], want[2]), ("dweight", dw, theirs[3], want[3]),
                          ("dbias", db, theirs[4], want[4])):
        a, t, e = (v[:, keep] if v.dim() == 5 else v[keep] for v in (a, t, e))
        assert _nerr(a, e) <= max(3 * _nerr(t, e), 1e-6), f"{name}: {_nerr(a, e):.3e} (torch fp32 {_nerr(t, e):.3e})"


# ------------------------------------------------------------------------------------------------------------------------------
# D: non-finite values against torch
# ------------------------------------------------------------------------------------------------------------------------------
def _torch_act(x, w, b, rm, rv, r, gy, training, relu, eps, dtype):
    xi = x.detach().to(dtype).clone().requires_grad_(True)
    wi = w.to(dtype).clone().requires_grad_(True) if w is not None else None
    bi = b.to(dtype).clone().requires_grad_(True) if b is not None else None
    y = F.batch_norm(xi, rm.to(dtype).clone(), rv.to(dtype).clone(), wi, bi, training, 0.1, eps)
    y = F.relu(y) if relu else y
    y = y + r.to(dtype) if r is not None else y
    y.backward(gy.to(dtype))
    return y.detach(), xi.grad, wi.grad if wi is not None else None, bi.grad if bi is not None else None


def _same_nonfinite(a, e, what):
    a, e = a.double(), e.double()
    assert torch.equal(a.isnan(), e.isnan()), f"{what}: NaN at {(a.isnan() != e.isnan()).nonzero()[:4].tolist()}"
    assert torch.equal(a == float("inf"), e == float("inf")) and torch.equal(a == -float("inf"), e == -float("inf")), f"{what}: inf"


def _finite_err(a, e):
    m = e.isfinite()
    return _nerr(a.double()[m], e.double()[m]) if bool(m.any()) else 0.0


@pytest.mark.parametrize("relu,residual,affine", list(itertools.product([True, False], repeat=3)), ids=str)
def test_eval_nonfinite_pixels_against_torch(relu, residual, affine):
    shape = (2, 5, 3, 9, 11)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(shape, generator=g)
    gy = torch.randn(shape, generator=g)
    r = torch.randn(shape, generator=g)
    for t, vals in ((x, (float("nan"), float("inf"), -float("inf"))), (gy, (float("nan"), float("inf"))), (r, (float("nan"), -float("inf")))):
        flat = t.view(-1)
        idx = torch.randperm(flat.numel(), generator=g)[:12]
        for k, i in enumerate(idx.tolist()):
            flat[i] = vals[k % len(vals)]
    x, gy, r = x.to(DEV), gy.to(DEV), (r.to(DEV) if residual else None)
    w = torch.tensor([1.0, -0.5, 2.0, 0.0, 0.7], device=DEV) if affine else None
    b = torch.tensor([0.1, 0.2, -0.3, 0.5, 0.0], device=DEV) if affine else None
    rm, rv = torch.randn(5, generator=g).to(DEV), (torch.rand(5, generator=g) + 0.5).to(DEV)
    y, mean, var = bn_forward(x, w, b, rm, rv, r, False, 1e-5, relu)
    dx, dw, db = bn_backward(gy, x, w, b, mean, var, False, 1e-5, relu, True, affine, affine)
    want = _torch_act(x, w, b, rm, rv, r, gy, False, relu, 1e-5, torch.float64)
    theirs = _torch_act(x, w, b, rm, rv, r, gy, False, relu, 1e-5, torch.float32)
    for name, a, t, e in zip(("y", "dx", "dweight", "dbias"), (y, dx, dw, db), theirs, want):
        if e is None:
            continue
        _same_nonfinite(a, e, name)
        assert _finite_err(a, e) <= max(3 * _finite_err(t, e), 1e-6), name


def test_training_nan_channel_against_torch():
    shape = (2, 6, 3, 40, 50)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(shape, generator=g).to(DEV)
    gy = torch.randn(shape, generator=g).to(DEV)
    w = (torch.rand(6, generator=g) + 0.5).to(DEV)
    b = (torch.rand(6, generator=g) - 0.5).to(DEV)
    clean = [*bn_forward(x, w, b, None, None, None, True, 1e-5, True)]
    clean += [*bn_backward(gy, x, w, b, clean[1], clean[2], True, 1e-5, True, True, True, True)]
    c = 3
    xn = x.clone()
    xn[1, c, 2, 17, 33] = float("nan")
    got = [*bn_forward(xn, w, b, None, None, None, True, 1e-5, True)]
    got += [*bn_backward(gy, xn, w, b, got[1], got[2], True, 1e-5, True, True, True, True)]
    y, mean, var, dx, dw, db = got
    assert bool(mean[c].isnan()) and bool(var[c].isnan()) and bool(y[:, c].isnan().all())
    want = _torch_act(xn, w, b, torch.zeros(6, device=DEV), torch.ones(6, device=DEV), None, gy, True, True, 1e-5, torch.float64)
    theirs = _torch_act(xn, w, b, torch.zeros(6, device=DEV), torch.ones(6, device=DEV), None, gy, True, True, 1e-5, torch.float32)
    assert bool(want[3][c].isfinite()) and bool(db[c].isfinite())
    err, err_t = abs(float(db[c]) - float(want[3][c])), abs(float(theirs[3][c]) - float(want[3][c]))
    assert err <= max(3 * err_t, 1e-6 * abs(float(want[3][c]))), (err, err_t)
    others = [i for i in range(6) if i != c]
    for name, a, e in zip(("y", "mean", "var", "dx", "dweight", "dbias"), got, clean):
        sel = (slice(None), others) if a.dim() == 5 else (others,)
        assert torch.equal(a[sel], e[sel]), name


# ------------------------------------------------------------------------------------------------------------------------------
# E: layouts and host routes
# ------------------------------------------------------------------------------------------------------------------------------
def _all(x, w, b, r, gy, training=True, relu=True, rm=None, rv=None, eps=1e-5):
    y, mean, var = bn_forward(x, w, b, rm, rv, r, training, eps, relu)
    dx, dw, db = bn_backward(gy, x, w, b, mean, var, training, eps, relu, True, True, True)
    return y, mean, var, dx, dw, db


def _equal(got, ref, what):
    for name, a, e in zip(("y", "mean", "var", "dx", "dw", "db"), got, ref):
        assert torch.equal(a, e), f"{what}: {name}"


def _layout_data(shape, seed):
    g = torch.Generator().manual_seed(seed)
    c = shape[1]
    return (torch.randn(shape, generator=g).to(DEV), (torch.rand(c, generator=g) + 0.5).to(DEV), (torch.rand(c, generator=g) - 0.5).to(DEV),
            torch.randn(shape, generator=g).to(DEV), torch.randn(shape, generator=g).to(DEV))


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_expanded_sliced_and_frame_major_inputs(training):
    b, c, s, X, Y = 2, 5, 3, 7, 600                                  # 4200 pixels: a whole piece and a short one
    _, w, bias, r, gy = _layout_data((b, c, s, X, Y), 1)
    rm, rv = torch.randn(c, device=DEV), torch.rand(c, device=DEV) + 0.5
    g = torch.Generator().manual_seed(2)
    views = {
        "b": TC.poisoned(torch.randn(1, c, s, X, Y, generator=g), DEV).expand(b, c, s, X, Y),
        "s": TC.poisoned(torch.randn(b, c, 1, X, Y, generator=g), DEV).expand(b, c, s, X, Y),
        "c": TC.poisoned(torch.randn(b, 1, s, X, Y, generator=g), DEV).expand(b, c, s, X, Y),
        "bs": TC.poisoned(torch.randn(1, c, 1, X, Y, generator=g), DEV).expand(b, c, s, X, Y),
    }
    big = TC.poisoned(torch.randn(b, c + 7, s, X, Y, generator=g), DEV)
    views["channel slice"] = big[:, 4:4 + c]                          # temporal_entry's outputs as norm_act receives them
    views["frame major"] = TC.poisoned_frame_major(torch.randn(b, c, s, X, Y, generator=g), DEV)
    for name, xv in views.items():
        assert not xv.is_contiguous()
        ref = _all(xv.contiguous(), w, bias, r, gy, training, True, rm, rv)
        _equal(_all(xv, w, bias, r, gy, training, True, rm, rv), ref, name)


def _shifted(t, by):
    """t's values at an address `by` floats past a 16-byte boundary"""
    buf = torch.full((t.numel() + 8,), float("nan"), device=DEV)
    v = buf[by:by + t.numel()].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_misaligned_pointers_in_every_combination(training):
    """x, residual, dy, y and dx each on or one float off a 16-byte boundary: every (vx, vy, vr), (vx, vg) and (vx, vg, vo) the apply
    and gradient passes branch on"""
    shape = (2, 3, 2, 1, 4100)
    x, w, b, r, gy = _layout_data(shape, 3)
    rm, rv = torch.randn(3, device=DEV), torch.rand(3, device=DEV) + 0.5
    for relu in (True, False):
        ref_y, ref_m, ref_v = abi_forward(x, w, b, rm, rv, r, training, relu, 1e-5)
        ref_g = abi_backward(x, gy, w, b, ref_m, ref_v, training, relu, 1e-5)
        for ox, orr, oy in itertools.product((0, 1), repeat=3):
            xs, rs = _shifted(x, ox), _shifted(r, orr)
            d = _desc(xs, training, relu, 1e-5)
            ws = _lib.workspace(_lib.load().fiery_batch_norm_workspace_bytes(d), DEV)
            ybuf = torch.full((x.numel() + 8,), float("nan"), device=DEV)
            y = ybuf[oy:oy + x.numel()]
            mean, var = torch.empty(3, device=DEV), torch.empty(3, device=DEV)
            _lib.call("fiery_batch_norm_forward", DEV, d, xs.data_ptr(), w.data_ptr(), b.data_ptr(), rm.data_ptr(), rv.data_ptr(),
                      rs.data_ptr(), y.data_ptr(), mean.data_ptr(), var.data_ptr(), ws.data_ptr())
            assert torch.equal(y.view(ref_y.shape), ref_y) and torch.equal(mean, ref_m) and torch.equal(var, ref_v), (ox, orr, oy)
        for ox, og, oo in itertools.product((0, 1), repeat=3):
            xs, gs = _shifted(x, ox), _shifted(gy, og)
            d = _desc(xs, training, relu, 1e-5)
            ws = _lib.workspace(_lib.load().fiery_batch_norm_workspace_bytes(d), DEV)
            dbuf = torch.full((x.numel() + 8,), float("nan"), device=DEV)
            dx = dbuf[oo:oo + x.numel()]
            dw, db = torch.empty(3, device=DEV), torch.empty(3, device=DEV)
            _lib.call("fiery_batch_norm_backward", DEV, d, xs.data_ptr(), gs.data_ptr(), w.data_ptr(), b.data_ptr(), ref_m.data_ptr(),
                      ref_v.data_ptr(), dx.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr())
            assert torch.equal(dx.view(ref_g[0].shape), ref_g[0]) and torch.equal(dw, ref_g[1]) and torch.equal(db, ref_g[2]), (ox, og, oo)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_half_inputs_directly_and_under_autocast(dtype):
    shape = (2, 6, 3, 9, 13)
    x, w, b, r, gy = _layout_data(shape, 4)
    xh, rh = x.to(dtype), r.to(dtype)
    ref = _all(xh.float(), w, b, rh.float(), gy)
    y, mean, var = bn_forward(xh, w, b, None, None, rh, True, 1e-5, True)
    assert torch.equal(y, ref[0]) and torch.equal(mean, ref[1]) and torch.equal(var, ref[2])
    dx, dw, db = bn_backward(gy, xh, w, b, mean, var, True, 1e-5, True, True, True, True)
    assert torch.equal(dx, ref[3]) and torch.equal(dw, ref[4]) and torch.equal(db, ref[5])
    xi = xh.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=dtype):
        ya, _, _ = torch.ops.fiery_b200.batch_norm_act(xi, w, b, None, None, rh, True, 1e-5, True)
    assert ya.dtype == torch.float32 and torch.equal(ya.detach(), ref[0])
    ya.backward(gy)
    assert xi.grad.dtype == dtype and torch.equal(xi.grad, ref[3].to(dtype))


def test_expanded_grad_and_strided_residual():
    shape = (2, 6, 3, 9, 13)
    x, w, b, r, _ = _layout_data(shape, 5)
    rs = TC.poisoned_frame_major(r, DEV)                              # a non-contiguous residual
    assert not rs.is_contiguous()
    ones = torch.ones(shape, device=DEV)
    ref = _all(x, w, b, r, ones)
    xi, wi, bi = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y, _, _ = torch.ops.fiery_b200.batch_norm_act(xi, wi, bi, None, None, rs, True, 1e-5, True)
    assert torch.equal(y.detach(), ref[0])
    y.sum().backward()                                                # grad_y: an expanded (stride-0) tensor of ones
    assert torch.equal(xi.grad, ref[3]) and torch.equal(wi.grad, ref[4]) and torch.equal(bi.grad, ref[5])


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_every_backward_subset_through_the_abi(training):
    shape = (2, 5, 3, 1, 4099)
    x, w, b, _, gy = _layout_data(shape, 6)
    rm, rv = torch.randn(5, device=DEV), torch.rand(5, device=DEV) + 0.5
    _, mean, var = abi_forward(x, w, b, rm, rv, None, training, True, 1e-5)
    full = abi_backward(x, gy, w, b, mean, var, training, True, 1e-5)
    for need in itertools.product((True, False), repeat=3):
        got = abi_backward(x, gy, w, b, mean, var, training, True, 1e-5, need)
        for k, a, e in zip(need, got, full):
            assert (a is None) != k and (a is None or torch.equal(a, e)), need


# ------------------------------------------------------------------------------------------------------------------------------
# F: the module over several steps
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(), dict(momentum=None), dict(track_running_stats=False), dict(affine=False)],
                         ids=["momentum0.1", "cumulative", "untracked", "no-affine"])
def test_module_over_several_steps_against_fp64(kw):
    torch.manual_seed(0)
    c = 7
    ref64 = nn.BatchNorm3d(c, **kw).to(DEV).double()
    if ref64.affine:
        with torch.no_grad():
            ref64.weight.copy_(torch.tensor([1.0, -0.5, 2.0, 0.0, 0.7, 1.3, -1.1]))
            ref64.bias.copy_(torch.tensor([0.1, 0.2, -0.3, 0.5, 0.0, -0.1, 0.4]))
    ref32 = copy.deepcopy(ref64).float()
    mine = FusedBatchNorm3d(copy.deepcopy(ref32))
    g = torch.Generator().manual_seed(1)
    shapes = [(2, c, 3, 20, 30), (1, c, 2, 64, 65), (3, c, 1, 5, 7), (2, c, 3, 1, 4097)]
    for step, shape in enumerate(shapes + [shapes[0]]):
        if step == len(shapes):
            for m in (ref64, ref32, mine):
                m.eval()
        x = (torch.randn(shape, generator=g) * (step + 1) + step).to(DEV)
        gy = torch.randn(shape, generator=g).to(DEV)
        outs = []
        for m, dt in ((ref64, torch.float64), (ref32, torch.float32), (mine, torch.float32)):
            m.zero_grad()
            xi = x.to(dt).requires_grad_(True)
            y = m(xi)
            y.backward(gy.to(dt))
            outs.append([y.detach(), xi.grad] + ([m.weight.grad, m.bias.grad] if m.affine else []))
        for name, e, t, a in zip(("y", "dx", "dweight", "dbias"), *outs):
            assert _nerr(a, e) <= max(3 * _nerr(t, e), 1e-6), f"step {step} {name}: {_nerr(a, e):.3e} (torch {_nerr(t, e):.3e})"
        for (n, a), (_, e) in zip(mine.named_buffers(), ref64.named_buffers()):
            if a.dtype.is_floating_point:
                assert _nerr(a, e) <= 1e-6, f"step {step} {n}: {_nerr(a, e):.3e}"
            else:
                assert torch.equal(a.cpu(), e.cpu()), n


# ------------------------------------------------------------------------------------------------------------------------------
# G: one whole TemporalModel at the shipped grid
# ------------------------------------------------------------------------------------------------------------------------------
def test_whole_model_at_the_shipped_grid():
    grid = (200, 200)
    ref = _model(3, 0, seed=3, grid=grid)
    sw = _swapped(ref, "all")
    ref64 = copy.deepcopy(ref).double()
    for m in (ref, sw, ref64):
        m.train(True)
    gen = torch.Generator().manual_seed(17)
    bev = torch.randn((2, 3, 64, *grid), generator=gen).to(DEV)
    ego = torch.randn((2, 3, 6), generator=gen).to(DEV)
    gout = torch.randn((2, 1, 64, *grid), generator=gen).to(DEV)
    y64, gx64, gp64 = _step(ref64, bev.double(), ego.double(), gout.double(), "concat")
    y0, gx0, gp0 = _step(ref, bev, ego, gout, "concat", tf32=True)
    y1, gx1, gp1 = _step(sw, bev, ego, gout, "folded")
    assert set(gp1) == set(gp0) == set(gp64)
    for what, a, r, o in [("out", y1, y64, y0), ("grad_bev", gx1, gx64, gx0)] + [(n, gp1[n], gp64[n], gp0[n]) for n in gp64]:
        err, bar = _nerr(a, r), max(3 * _nerr(o, r), 1e-5)
        assert err <= bar, f"{what}: {err:.3e} vs oracle {_nerr(o, r):.3e}"
    for (n, b1), (_, b0) in zip(sw.named_buffers(), ref.named_buffers()):
        if b1.dtype.is_floating_point:
            assert _nerr(b1, b0) < 1e-3, n
        else:
            assert torch.equal(b1, b0), n
