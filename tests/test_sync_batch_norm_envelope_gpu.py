"""GPU: batch statistics over a process group (fiery_batch_norm_local_stats / _forward_gathered / _local_grad_sums /
_backward_gathered, FusedSyncBatchNorm, the SpatialGRU's step entries) across the rank splits of tests/_batch_norm_cases.py, with
simulated ranks in one process (a ``torch.stack`` of the ranks' triplets standing in for the gather) unless said otherwise.

A  exact group cases bit for bit against ``restate_group`` through the C ABI, every ``SPLITS`` entry and both exact variants (equal
   rank means; rank means apart, the cross-rank delta^2 term exact): NaN-poisoned inputs, outputs between sentinel margins, workspaces
   of exactly the sync size, NULL count_out, NULL dgamma / dbeta and NULL pointers for empty ranks;
B  random data bit for bit where the restatement is exact: the group mean (plain or contracted fp64), the count, each rank's dbeta,
   y = fmaf(scale, x, shift) from the kernel's own statistics, the same bits on every rank, and a group with one non-empty rank bit
   for bit the single-rank operators at every position of that rank;
C  every element against fp64 on the whole batch given the kernel's statistics, the statistics per channel and the outputs normwise
   within 3x torch's own SyncBatchNorm arithmetic, across BNC.SHAPE_LIST x SPLITS and hard statistics across ranks;
D  NaN and +-inf on one rank poison that channel's statistics on every rank;
E  the module route (FusedSyncBatchNorm with a fake gather) bit for bit the contiguous fp32 phases: half inputs, strided and sliced x,
   an expanded grad_y, a residual of another dtype, 2-D to 4-D inputs, momentum=None, affine=False, track_running_stats=False, and
   inputs with no elements of every shape;
F  the SpatialGRU's step entries through the C ABI at worlds 2 to 4 with an empty rank 0, every output on guarded buffers, every stage
   and gradient element by element, the same bits as the module's step generators;
G  three processes on one GPU over gloo, rank 0 empty, one gather per norm call and per GRU step each way on every rank."""
from __future__ import annotations

import copy
import datetime
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from fiery_b200 import _lib
from fiery_b200 import batch_norm as BN
from fiery_b200._lib import f32_planes
from tests import _batch_norm_cases as BC
from tests import _spatial_gru_cases as gc
from tests import _temporal_cases as TC

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EPS = 1e-5
MARGINS = {}                     # output -> the largest err / bound seen, reported at the end of the module
_ids = lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v)     # noqa: E731


@pytest.fixture(scope="module", autouse=True)
def _report_margins():
    yield
    if MARGINS:
        print("\nlargest err/bound per output: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(MARGINS.items())))


def _note(name, r):
    MARGINS[name] = max(MARGINS.get(name, 0.0), r)


def _np(t):
    return t.detach().cpu().numpy()


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# the group entries through the C ABI on guarded buffers
# ------------------------------------------------------------------------------------------------------------------------------
def _desc(shape, relu, eps):
    b, c, s, p = shape
    d = _lib.BatchNormDesc()
    d.batch, d.channels, d.frames, d.pixels = b, c, s, p
    d.stride_b, d.stride_c, d.stride_t = c * s * p, s * p, p
    d.training, d.relu, d.eps = 1, int(relu), float(eps)
    return d


def _guarded(n, dtype=torch.float32):
    """(buffer, view) of n NaN elements between sentinel margins; fp64 ones as a float32 buffer twice as long"""
    words = 2 * n if dtype == torch.float64 else n
    buf, view = TC.guarded(words, 64, 64, DEV)
    return buf, (view.view(torch.float64) if dtype == torch.float64 else view)


class _Outs:
    """every guarded output of a call, checked to be written (where asked) and contained"""

    def __init__(self):
        self.items = []

    def __call__(self, n, what, dtype=torch.float32, must_write=True):
        buf, view = _guarded(n, dtype)
        self.items.append((buf, view, what, must_write))
        return view

    def check(self, finite=True):
        """finite: every element asked for was written with a number (an fp64 one checked as fp64)"""
        torch.cuda.synchronize()
        for buf, view, what, must in self.items:
            wide = view.dtype == torch.float64
            TC.assert_written_and_contained(buf, view.view(torch.float32) if wide else view, what,
                                            must_write=finite and must and not wide and view.numel() > 0)
            if finite and must and wide:
                assert not bool(_unwritten(view).any()), f"{what}: never written"


def _unwritten(view):
    """per element, whether it still holds the fill: two NaN words (an fp64 element) or a NaN"""
    return view.view(torch.float32).view(-1, 2).isnan().all(1) if view.dtype == torch.float64 else view.isnan()


def _untouched(view, what):
    assert bool(_unwritten(view).all()), f"{what}: a NULL output's buffer was written"


def _workspace(d, outs, what):
    nbytes = int(_lib.load().fiery_batch_norm_sync_workspace_bytes(d))
    assert nbytes > 0 and nbytes % 4 == 0
    return outs(nbytes // 4, what, must_write=False)


def abi_group(shards, w, b, rs, dys, relu, eps, null_count=False, null_params=False, finite=True):
    """The four group entries for every rank of ``shards`` (numpy (b_r, C, s, pixels), b_r may be 0) from NaN-poisoned inputs into
    guarded outputs; an empty rank passes NULL x / y / residual / grad_y / grad_x.  Returns the dict ``restate_group`` returns."""
    c = shards[0].shape[1]
    wt, bt = _t(w), _t(b)
    ptr = lambda t: 0 if t is None or t.numel() == 0 else t.data_ptr()         # noqa: E731
    xs = [TC.poisoned(torch.from_numpy(x), DEV) if x.size else None for x in shards]
    rt = [TC.poisoned(torch.from_numpy(r), DEV) if r is not None and r.size else None for r in rs]
    gt = [TC.poisoned(torch.from_numpy(g), DEV) if g.size else None for g in dys]
    outs = _Outs()
    stats = []
    for x, xn in zip(xs, shards):
        d = _desc(xn.shape, relu, eps)
        st = outs(3 * c, "local stats", torch.float64)
        _lib.call("fiery_batch_norm_local_stats", DEV, d, ptr(x), st.data_ptr(), _workspace(d, outs, "local stats workspace").data_ptr())
        stats.append(st.view(c, 3))
    gathered = torch.stack(stats)
    res = dict(mean=[], var=[], count=[], y=[], dx=[], dw=[], db=[], gathered_forward=gathered, sums=[])
    for x, xn, r in zip(xs, shards, rt):
        d = _desc(xn.shape, relu, eps)
        y = outs(xn.size, "y")
        mean, var = outs(c, "mean"), outs(c, "var")
        count = outs(1, "count", torch.float64, must_write=not null_count)
        _lib.call("fiery_batch_norm_forward_gathered", DEV, d, len(shards), gathered.data_ptr(), ptr(x), ptr(wt), ptr(bt), ptr(r), ptr(y),
                  mean.data_ptr(), var.data_ptr(), 0 if null_count else count.data_ptr(), _workspace(d, outs, "forward workspace").data_ptr())
        if null_count:
            torch.cuda.synchronize()
            _untouched(count, "count_out")
        for k, v in (("y", y.view(xn.shape)), ("mean", mean), ("var", var), ("count", count)):
            res[k].append(v)
    for x, xn, g, mean, var in zip(xs, shards, gt, res["mean"], res["var"]):
        d = _desc(xn.shape, relu, eps)
        sums = outs(3 * c, "sums", torch.float64)
        dw, db = outs(c, "dweight", must_write=not null_params), outs(c, "dbias", must_write=not null_params)
        _lib.call("fiery_batch_norm_local_grad_sums", DEV, d, ptr(x), ptr(g), ptr(wt), ptr(bt), mean.data_ptr(), var.data_ptr(),
                  sums.data_ptr(), 0 if null_params else ptr(dw), 0 if null_params else ptr(db),
                  _workspace(d, outs, "grad sums workspace").data_ptr())
        if null_params:
            torch.cuda.synchronize()
            _untouched(dw, "dweight")
            _untouched(db, "dbias")
        res["sums"].append(sums.view(c, 3))
        res["dw"].append(dw)
        res["db"].append(db)
    gathered_b = torch.stack(res["sums"])
    for x, xn, g, mean, var in zip(xs, shards, gt, res["mean"], res["var"]):
        d = _desc(xn.shape, relu, eps)
        dx = outs(xn.size, "dx")
        _lib.call("fiery_batch_norm_backward_gathered", DEV, d, len(shards), gathered_b.data_ptr(), ptr(x), ptr(g), ptr(wt), ptr(bt),
                  mean.data_ptr(), var.data_ptr(), ptr(dx), _workspace(d, outs, "backward workspace").data_ptr())
        res["dx"].append(dx.view(xn.shape))
    outs.check(finite)
    res["gathered_backward"] = gathered_b
    return res


def _same_on_every_rank(res):
    for k in ("mean", "var", "count"):
        for v in res[k][1:]:
            assert torch.equal(v, res[k][0]) or (k == "count" and bool(v.isnan().all())), k


# ------------------------------------------------------------------------------------------------------------------------------
# A: exact group cases, bit for bit
# ------------------------------------------------------------------------------------------------------------------------------
def _exact_shape(name):
    return (2, 3, 1, 1, 1) if name == "1+1" else (8, 3, 1, 1, 4097)


def _run_exact(case, relu, null_count, null_params):
    sizes = case["sizes"]
    x, r, dy = (BC.shards_of(case[k], sizes) for k in ("x", "r", "dy"))
    got = abi_group(x, case["w"], case["b"], r, dy, relu, case["eps"], null_count, null_params)
    want = BC.restate_group(x, case["w"], case["b"], r, dy, relu, case["eps"])
    _same_on_every_rank(got)
    for k, (xk, mean, var, count) in enumerate(zip(x, got["mean"], got["var"], got["count"])):
        assert _bits_equal(_np(mean), want["mean"]) and _bits_equal(_np(var), want["var"]), k
        if not null_count:
            assert float(count) == float(want["count"][0]) == case["x"].size // case["x"].shape[1], k
    for name in ("y", "dx") + (() if null_params else ("dw", "db")):
        for k, (a, e) in enumerate(zip(got[name], want[name])):
            assert _bits_equal(_np(a), e), f"{sizes} rank {k} {name}: {np.abs(_np(a).astype(np.float64) - e).max():.3e}"
    return got, want


@pytest.mark.parametrize("name", BC.SPLIT_NAMES)
def test_exact_every_split(name):
    shape = _exact_shape(name)
    sizes = BC.split_sizes(name, shape[0])
    case = BC.exact_group_case(shape, sizes, seed=len(sizes))
    k = BC.SPLIT_NAMES.index(name)
    _run_exact(case, True, null_count=k % 2 == 1, null_params=k % 3 == 2)
    _run_exact(case, False, null_count=False, null_params=False)


@pytest.mark.parametrize("shape,sizes", [((8, 5, 2, 1, 6), [0, 1, 0, 1, 2, 4]), ((16, 3, 1, 1, 4100), [2, 2, 4, 0, 8]),
                                         ((8, 4, 3, 40, 50), [1, 1, 2, 4]), ((8, 2, 1, 1, 8193), [0, 0, 1, 1, 2, 4, 0])], ids=str)
def test_exact_rank_means_apart(shape, sizes):
    """the ranks' means differ by integers: Chan's cross-rank delta^2 term non-zero and exact"""
    case = BC.exact_group_case(shape, sizes, seed=5, offsets=True)
    got, want = _run_exact(case, True, False, False)
    trip = _np(got["gathered_forward"])
    assert len({float(t[0, 1]) for t in trip if t[0, 0]}) > 1
    assert np.array_equal(_np(got["mean"][0]), case["mu"].astype(np.float32)) and np.all(_np(got["var"][0]) == case["var"])


# ------------------------------------------------------------------------------------------------------------------------------
# B: random data, bit for bit where the restatement is exact
# ------------------------------------------------------------------------------------------------------------------------------
def _random(shape, seed, spread=4.0):
    rng = np.random.default_rng(seed)
    b, c, s, X, Y = shape
    p = X * Y
    x = (rng.standard_normal((b, c, s, p)) * np.exp2(rng.integers(-3, 4, (b, c, s, p))) +
         rng.standard_normal((b, c, 1, 1)) * spread).astype(np.float32)
    w = (rng.standard_normal(c) * 1.5).astype(np.float32)
    w[::5] = -np.abs(w[::5])
    bias = rng.standard_normal(c).astype(np.float32)
    r = rng.standard_normal((b, c, s, p)).astype(np.float32)
    dy = rng.standard_normal((b, c, s, p)).astype(np.float32)
    return x, w, bias, r, dy


def _either(got, a, b_):
    """per channel, got's bits are a's or b_'s (the plain or the contracted fp64 arithmetic)"""
    got, a, b_ = (np.asarray(t, np.float32).view(np.int32) for t in (got, a, b_))
    return np.flatnonzero(~((got == a) | (got == b_)))


B_CASES = [((4, 35, 1, 1, 4093), "1+rest"), ((8, 6, 2, 1, 4100), "8:3empty"), ((4, 3, 1, 64, 64), "0+0+a+b"),
           ((6, 4, 3, 20, 20), "a+0+b+0"), ((40, 5, 1, 1, 7), "64"), ((3, 129, 2, 1, 5), "0x5+all")]


@pytest.mark.parametrize("shape,name", B_CASES, ids=str)
def test_random_data_against_the_restatement(shape, name):
    x, w, bias, r, dy = _random(shape, sum(shape))
    sizes = BC.split_sizes(name, shape[0])
    xs, rs, dys = (BC.shards_of(t, sizes) for t in (x, r, dy))
    for relu, residual in ((True, False), (False, True)):
        got = abi_group(xs, w, bias, rs if residual else [None] * len(sizes), dys, relu, EPS)
        _same_on_every_rank(got)
        plain, contracted = (BC.restate_group(xs, w, bias, rs, dys, relu, EPS, k) for k in (False, True))
        mean, var = _np(got["mean"][0]), _np(got["var"][0])
        bad = _either(mean, plain["mean"], contracted["mean"])
        assert bad.size == 0, f"mean of channels {bad[:8]}"
        assert float(got["count"][0]) == x.size // shape[1]
        scale, sh_u, sh_c = BC.scale_shift(w, bias, mean, var, EPS)
        for k, (xk, rk, dyk) in enumerate(zip(xs, rs, dys)):
            if not xk.size:
                continue
            yk = _np(got["y"][k])
            want = []
            for sh in (sh_u, sh_c):
                pre = BC.fmaf_exact(scale.reshape(1, -1, 1, 1), xk, sh.reshape(1, -1, 1, 1))
                yy = np.where(pre < 0, np.float32(0), pre) if relu else pre
                want.append((yy + rk).astype(np.float32) if residual else yy)
            bad = np.flatnonzero(~np.all((yk.view(np.int32) == want[0].view(np.int32)) | (yk.view(np.int32) == want[1].view(np.int32)),
                                         axis=(0, 2, 3)))
            assert bad.size == 0, f"rank {k} y of channels {bad[:8]}"
            if not residual:                                            # dbeta: the rank's own fp64 sum of its pieces' sums of g'
                g = np.where(yk > 0, dyk, np.float32(0)) if relu else dyk
                p = xk.shape[-1]
                want_db = BC.seq_sum64(BC.channel_pieces(BC.bn_piece_sums_model(g, p), p)).astype(np.float32)
                assert _bits_equal(_np(got["db"][k]), want_db), f"rank {k} dbias"


@pytest.mark.parametrize("name", ["1+rest", "8:3empty", "0+0+a+b", "a+0+b+0"])
def test_cancelling_means_show_the_merge_order(name):
    """the group's mean is exactly 0, so the fp32 mean is the rank merge's fp64 rounding residue: ascending order, plain or
    contracted, and nothing else"""
    x = BC.cancelling_case(64, 1)
    sizes = BC.split_sizes(name, x.shape[0])
    xs = BC.shards_of(x, sizes)
    zeros = [np.zeros_like(t) for t in xs]
    got = abi_group(xs, None, None, [None] * len(sizes), zeros, False, EPS)
    plain, contracted = (BC.restate_group(xs, None, None, [None] * len(sizes), zeros, False, EPS, k) for k in (False, True))
    bad = _either(_np(got["mean"][0]), plain["mean"], contracted["mean"])
    assert bad.size == 0, f"mean of channels {bad[:8]}: {_np(got['mean'][0])[bad[:4]]} vs {plain['mean'][bad[:4]]}"


@pytest.mark.parametrize("world", [2, 4])
def test_one_non_empty_rank_is_the_single_rank_operator(world):
    shape = (3, 35, 2, 33, 130)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(shape, generator=g).to(DEV) * 3 + 1
    dy, r = torch.randn(shape, generator=g).to(DEV), torch.randn(shape, generator=g).to(DEV)
    w, b = (1 + 0.3 * torch.randn(35, generator=g)).to(DEV), (0.3 * torch.randn(35, generator=g)).to(DEV)
    y0, m0, v0 = torch.ops.fiery_b200.batch_norm_act(x, w, b, None, None, r, True, EPS, True)
    dx0, dw0, db0 = torch.ops.fiery_b200.batch_norm_act_backward(dy, x, w, b, m0, v0, True, EPS, True, True, True, True)
    empty = x[:0]
    for at in range(world):
        xs = [x if k == at else empty for k in range(world)]
        stats = torch.stack([BN.local_stats(f32_planes(t)) for t in xs])
        fw = [BN.forward_gathered(stats, t, w, b, r if k == at else r[:0], EPS, True) for k, t in enumerate(xs)]
        sums = [BN.local_grad_sums(dy if k == at else dy[:0], t, w, b, f[1], f[2], EPS, True, True, True) for k, (t, f) in
                enumerate(zip(xs, fw))]
        gb = torch.stack([s[0] for s in sums])
        dx = BN.backward_gathered(gb, dy, x, w, b, fw[at][1], fw[at][2], EPS, True)
        for f in fw:
            assert torch.equal(f[1], m0) and torch.equal(f[2], v0) and float(f[3]) == x.numel() // 35
        assert torch.equal(fw[at][0], y0) and torch.equal(dx, dx0), at
        assert torch.equal(sums[at][1], dw0) and torch.equal(sums[at][2], db0), at


# ------------------------------------------------------------------------------------------------------------------------------
# C: every element against fp64, the statistics and the norms against torch's SyncBatchNorm arithmetic
# ------------------------------------------------------------------------------------------------------------------------------
def _torch_sync(shards, w, b, rs, dys, relu, eps):
    """torch's SyncBatchNorm arithmetic in one process on the device in fp32: batch_norm_stats per non-empty shard,
    batch_norm_gather_stats_with_counts, batch_norm_elemt, batch_norm_backward_reduce, the sums added over the ranks, and
    batch_norm_backward_elemt.  Returns (y, dx) on the whole batch, mean and biased var."""
    full = [k for k, s in enumerate(shards) if s.numel()]
    st = [torch.batch_norm_stats(shards[k], eps) for k in full]
    counts = torch.tensor([shards[k].numel() // shards[k].shape[1] for k in full], dtype=torch.float32, device=DEV)
    mean, invstd = torch.batch_norm_gather_stats_with_counts(shards[full[0]], torch.stack([s[0] for s in st]),
                                                             torch.stack([s[1] for s in st]), None, None, 0.0, eps, counts)
    ys, red = [], []
    for k in full:
        y = torch.batch_norm_elemt(shards[k], w, b, mean, invstd, eps)
        gy = dys[k] * (y > 0) if relu else dys[k]
        ys.append((torch.relu(y) if relu else y) + (rs[k] if rs[k] is not None else 0))
        red.append((y, gy, torch.batch_norm_backward_reduce(gy, shards[k], mean, invstd, w, True, False, False)))
    sum_dy = sum(t[2][0] for t in red)
    sum_dy_xmu = sum(t[2][1] for t in red)
    dx = [torch.batch_norm_backward_elemt(gy, shards[k], mean, invstd, w, sum_dy, sum_dy_xmu, counts.to(torch.int32))
          for k, (_, gy, _) in zip(full, red)]
    var = (1.0 / invstd.double() ** 2 - eps).float()
    return torch.cat(ys), torch.cat(dx), mean, var


def _nerr(a, e):
    a, e = a.double(), e.double()
    return float((a - e).norm() / e.norm().clamp_min(1e-300))


def _check_against_fp64(x, w, b, r, dy, sizes, relu, eps, label):
    c = x.shape[1]
    n = x.numel() // c
    xs, rs, dys = (list(torch.split(t, sizes)) if t is not None else [None] * len(sizes) for t in (x, r, dy))
    flat = lambda t: t.reshape(t.shape[0], c, t.shape[2], t.shape[3] * t.shape[4])  # noqa: E731
    got = abi_group([_np(flat(t)) for t in xs], _np(w), _np(b), [_np(flat(t)) if t is not None else None for t in rs],
                    [_np(flat(t)) for t in dys], relu, eps)
    _same_on_every_rank(got)
    mean, var = got["mean"][0].double(), got["var"][0].double()
    y, dx = torch.cat(got["y"]).view(x.shape).double(), torch.cat(got["dx"]).view(x.shape).double()
    x64, w64, b64, dy64 = x.double(), w.double(), b.double(), dy.double()
    bc = lambda v: v.view(1, -1, 1, 1, 1)                                          # noqa: E731
    mean64, var64 = x64.mean(dim=(0, 2, 3, 4)), x64.var(dim=(0, 2, 3, 4), unbiased=False)
    ty, tdx, tmean, tvar = _torch_sync([t.float() for t in xs], w, b, rs, dys, relu, eps)
    # the statistics per channel: within 3x torch's SyncBatchNorm error, or a few fp32 roundings of the exact value
    err, err_t = (var - var64).abs(), (tvar.double() - var64).abs()
    # the floor: the pieces' fp32 means are rounded, so Chan's deltas between pieces carry 2^-24 (|mu| + sigma) each
    floor = torch.where(var64 == 0, (2.0 ** -22 * mean64.abs()) ** 2, 8 * 2.0 ** -24 * (var64 + mean64.abs() * var64.sqrt()))
    assert bool((err <= torch.maximum(3 * err_t, floor)).all()), f"{label} var: {err.max():.3e} torch {err_t.max():.3e}"
    merr, merr_t = (mean - mean64).abs(), (tmean.double() - mean64).abs()
    assert bool((merr <= torch.maximum(3 * merr_t, 4 * 2.0 ** -24 * (mean64.abs() + var64.sqrt()))).all()), f"{label} mean"
    # every element of y against fp64 with the kernel's statistics: scale and shift rounded to fp32, then y's own rounding
    ve = var + eps
    scale64 = w64 / ve.sqrt()
    pre64 = bc(scale64) * (x64 - bc(mean)) + bc(b64)
    scale32, shift32 = bc(scale64.float().double()), bc((b64 - mean * scale64).float().double())
    y64 = (pre64.clamp_min(0) if relu else pre64) + (r.double() if r is not None else 0)
    bound = 2.0 ** -23 * ((scale32 * x64).abs() + shift32.abs()) + 2.0 ** -24 * y64.abs()
    if relu:                                                        # where the pre-activation is within its bound of 0 either side
        bound = bound + torch.where(pre64.abs() <= bound, pre64.abs(), torch.zeros_like(pre64))
    ratio = float(((y - y64).abs() / bound.clamp_min(1e-300)).max())
    _note("y", ratio)
    assert ratio <= 1.0, f"{label} y: err/bound {ratio:.3g}"
    # dx against fp64 with the kernel's statistics and the kernel's ReLU mask: the bound carries the fp32 piece sums' error
    assert r is None or not relu, "the ReLU mask is read from y: no residual"
    mask = y > 0 if relu else torch.ones_like(x64, dtype=torch.bool)
    gm = torch.where(mask, dy64, torch.zeros_like(dy64))
    dmu = x64 - bc(mean)
    s1, s2 = gm.sum(dim=(0, 2, 3, 4)), (gm * dmu).sum(dim=(0, 2, 3, 4))
    e1 = BC_SUM * 2.0 ** -24 * gm.abs().sum(dim=(0, 2, 3, 4))
    e2 = BC_SUM * 2.0 ** -24 * (gm * dmu).abs().sum(dim=(0, 2, 3, 4)) + 2.0 ** -24 * (gm.abs() * dmu.abs()).sum(dim=(0, 2, 3, 4))
    k1, k0 = -scale64 * s2 / (n * ve), -scale64 * s1 / n
    dx64 = bc(scale64) * gm + bc(k1) * dmu + bc(k0)
    dbound = 8 * 2.0 ** -24 * ((bc(scale64) * gm).abs() + (bc(k1) * dmu).abs() + bc(k0).abs()) + \
        bc(scale64.abs()) * (bc(e1) / n + dmu.abs() * bc(e2) / (n * bc(ve)))
    dratio = float(((dx - dx64).abs() / dbound.clamp_min(1e-300)).max())
    _note("dx", dratio)
    assert dratio <= 1.0, f"{label} dx: err/bound {dratio:.3g}"
    # each rank's dgamma, dbeta against its own fp64 sums
    for k, (gk, dk) in enumerate(zip(torch.split(gm, sizes), torch.split(dmu, sizes))):
        sdb, sdw = gk.sum(dim=(0, 2, 3, 4)), (gk * dk).sum(dim=(0, 2, 3, 4)) / ve.sqrt()
        eb = BC_SUM * 2.0 ** -24 * gk.abs().sum(dim=(0, 2, 3, 4)) + 2.0 ** -24 * sdb.abs()
        ew = (BC_SUM + 2) * 2.0 ** -24 * (gk * dk).abs().sum(dim=(0, 2, 3, 4)) / ve.sqrt() + 2.0 ** -24 * sdw.abs()
        for nm, a, e, bd in (("db", got["db"][k], sdb, eb), ("dw", got["dw"][k], sdw, ew)):
            rr = float(((a.double() - e).abs() / bd.clamp_min(1e-300)).max())
            _note(nm, rr)
            assert rr <= 1.0, f"{label} rank {k} {nm}: err/bound {rr:.3g}"
    # normwise, against torch's own SyncBatchNorm arithmetic
    ref_y = (bc(w64) * (x64 - bc(mean64)) / bc(var64 + eps).sqrt() + bc(b64))
    ref_y = (ref_y.clamp_min(0) if relu else ref_y) + (r.double() if r is not None else 0)
    # or the header's arithmetic: shift = beta - mean scale rounded to fp32 carries 2^-24 |mean scale|, which torch's
    # (x - mean) invstd does not
    floor = max(float((2.0 ** -23 * ((scale32 * x64).abs() + shift32.abs())).norm() / ref_y.norm()), 1e-6)
    assert _nerr(y, ref_y) <= max(3 * _nerr(ty, ref_y), floor), f"{label} y normwise {_nerr(y, ref_y):.3e} torch {_nerr(ty, ref_y):.3e}"
    # dx the same way, measured against the larger of |dx| and the scale g' its terms cancel from (a channel of two values has dx
    # near 0); the floor the per-element bound above, or 1e-6 (the single-rank envelope's convention)
    xh64 = (x64 - bc(mean64)) / bc(var64 + eps).sqrt()
    pre_ref = bc(w64) * xh64 + bc(b64)
    g64 = torch.where(pre_ref > 0, dy64, torch.zeros_like(dy64)) if relu else dy64
    dx_ref = bc(w64) / bc(var64 + eps).sqrt() * (g64 - bc(g64.mean(dim=(0, 2, 3, 4))) - xh64 * bc((g64 * xh64).mean(dim=(0, 2, 3, 4))))
    size = max(float(dx_ref.norm()), float((bc(w64) / bc(var64 + eps).sqrt() * g64).norm()), 1e-300)
    err, err_t = float((dx - dx_ref).norm()) / size, float((tdx.double() - dx_ref).norm()) / size
    assert err <= max(3 * err_t, float(dbound.norm()) / size, 1e-6), f"{label} dx normwise {err:.3e} torch {err_t:.3e}"
    return got


BC_SUM = 32                      # terms along the piece sums' blocked order (tests/_spatial_gru_cases.py BN_SUM), and the fp64 rest


@pytest.mark.parametrize("name", BC.SPLIT_NAMES)
@pytest.mark.parametrize("shape", BC.SHAPE_LIST, ids=_ids)
def test_every_element_against_fp64(shape, name):
    sizes = BC.split_sizes(name, shape[0])
    if sizes is None:
        pytest.skip(f"{name} needs another batch")
    g = torch.Generator().manual_seed(sum(shape) + len(sizes))
    c = shape[1]
    x = (torch.randn(shape, generator=g) * 2 + torch.randn(shape[0], c, 1, 1, 1, generator=g) * 3).to(DEV)
    dy = torch.randn(shape, generator=g).to(DEV)
    w, b = (1 + 0.5 * torch.randn(c, generator=g)).to(DEV), (0.3 * torch.randn(c, generator=g)).to(DEV)
    w[::4] *= -1
    if shape[0] * shape[2] * shape[3] * shape[4] < 2:
        pytest.skip("one value per channel")
    _check_against_fp64(x, w, b, None, dy, sizes, True, EPS, f"{shape} {name}")     # y > 0 is then the kernel's ReLU mask


HARD = [("far", 1e-5, "8:3empty"), ("far", 0.0, "1+rest"), ("flat", 0.1, "0+0+a+b"), ("far", 0.1, "a+0+b+0"), ("flat", 1e-5, "64")]


@pytest.mark.parametrize("kind,eps,name", HARD, ids=str)
def test_hard_statistics_across_ranks(kind, eps, name):
    """rank means 1e4 to 1e5 apart with sigma 1e-2 (the cross-rank delta^2 carries all the variance), a constant channel, gamma < 0
    and gamma = 0, eps 0 and 0.1"""
    shape = (8, 6, 1, 40, 50)
    g = torch.Generator().manual_seed(len(kind) + int(eps * 100))
    z = torch.randn(shape, generator=g, dtype=torch.float64)
    w = torch.tensor([1.0, -1.5, 0.0, 0.75, 2.0, -0.25], dtype=torch.float64)
    bias = torch.tensor([0.1, -0.2, 0.3, 0.0, -0.5, 0.25], dtype=torch.float64)
    if kind == "far":
        apart = torch.tensor([1e4, 3e4, 1e5, 1e4, 5e4, 2e4], dtype=torch.float64)
        offs = torch.tensor([(-1) ** k * (k + 1) for k in range(shape[0])], dtype=torch.float64)
        x = z * 1e-2 + offs.view(-1, 1, 1, 1, 1) * apart.view(1, -1, 1, 1, 1)
    else:
        x = z * torch.tensor([1.0, 1e-3, 0.0, 2.0, 0.0, 1e-2], dtype=torch.float64).view(1, -1, 1, 1, 1) + \
            torch.tensor([0.0, 5.0, 0.375, -1.0, 0.0, 0.0], dtype=torch.float64).view(1, -1, 1, 1, 1)
        bias[4] = 0.5
    dy = torch.randn(shape, generator=g)
    sizes = BC.split_sizes(name, shape[0])
    _check_against_fp64(x.float().to(DEV), w.float().to(DEV), bias.float().to(DEV), None, dy.to(DEV), sizes, True, eps,
                        f"{kind} {eps} {name}")


# ------------------------------------------------------------------------------------------------------------------------------
# D: NaN and +-inf on one rank
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value", [float("nan"), float("inf"), -float("inf")], ids=["nan", "inf", "-inf"])
def test_nonfinite_on_one_rank_poisons_its_channel_everywhere(value):
    shape = (6, 5, 2, 1, 4100)
    x, w, bias, r, dy = _random(shape, 4)
    sizes = BC.split_sizes("8:3empty", shape[0])
    clean = abi_group(BC.shards_of(x, sizes), w, bias, BC.shards_of(r, sizes), BC.shards_of(dy, sizes), True, EPS)
    c = 3
    xp = x.copy()
    xp[4, c, 1, 4097] = value                                       # on one rank, in a channel's second piece
    xs = BC.shards_of(xp, sizes)
    got = abi_group(xs, w, bias, BC.shards_of(r, sizes), BC.shards_of(dy, sizes), True, EPS, finite=False)
    want = BC.restate_group(xs, w, bias, BC.shards_of(r, sizes), BC.shards_of(dy, sizes), True, EPS, True)
    others = [k for k in range(shape[1]) if k != c]
    for k in range(len(sizes)):
        assert bool(got["mean"][k][c].isnan()) and bool(got["var"][k][c].isnan()), k
        assert torch.equal(got["mean"][k][others], clean["mean"][k][others]) and torch.equal(got["var"][k][others], clean["var"][k][others])
        yk = _np(got["y"][k])
        assert np.array_equal(np.isnan(yk), np.isnan(want["y"][k])), k
        assert bool(np.isnan(yk[:, c]).all()) or yk.size == 0
        assert np.array_equal(yk[:, others], _np(clean["y"][k])[:, others]), k
        assert np.array_equal(np.isnan(_np(got["dx"][k])), np.isnan(want["dx"][k])), k


# ------------------------------------------------------------------------------------------------------------------------------
# E: the module route with a fake gather, bit for bit the contiguous fp32 phases
# ------------------------------------------------------------------------------------------------------------------------------
def _phases(xs, w, b, rs, dys, relu):
    """the contiguous fp32 phase calls for every rank: (gathered forward, gathered backward, per-rank (y, mean, var, count, dx, dw, db))"""
    x5 = [f32_planes(t.float().contiguous()) for t in xs]
    gf = torch.stack([BN.local_stats(t) for t in x5])
    fw = [BN.forward_gathered(gf, t, w, b, r.float() if r is not None else None, EPS, relu) for t, r in zip(x5, rs)]
    sums = [BN.local_grad_sums(g.float().contiguous(), t, w, b, f[1], f[2], EPS, relu, w is not None, b is not None)
            for t, g, f in zip(x5, dys, fw)]
    gb = torch.stack([s[0] for s in sums])
    out = []
    for t, g, f, s in zip(x5, dys, fw, sums):
        dx = BN.backward_gathered(gb, g.float().contiguous(), t, w, b, f[1], f[2], EPS, relu)
        out.append((f[0], f[1], f[2], f[3], dx, s[1], s[2]))
    return gf, gb, out


def _module(c, **kw):
    torch.manual_seed(0)
    bn = nn.SyncBatchNorm(c, **kw).to(DEV).train()
    if bn.affine:
        with torch.no_grad():
            bn.weight.copy_(torch.linspace(-1.5, 2.0, c))
            bn.bias.copy_(torch.linspace(-0.3, 0.4, c))
    return BN.FusedSyncBatchNorm(bn)


def _drive(module, x, rank, gf, gb, relu, residual=None, grad=None):
    """module.forward_act on this rank, its two gathers answered with the group's triplets, this rank's own in its place"""
    calls = []

    def gather(t, group):
        calls.append(group)
        whole = (gf if len(calls) == 1 else gb).clone()
        assert torch.equal(t, whole[rank]), "the rank's own triplet differs from the contiguous fp32 call's"
        whole[rank] = t
        return whole
    old = BN.gather, BN.sync_group
    BN.gather, BN.sync_group = gather, (lambda norm: "group")
    try:
        xi = x.detach().requires_grad_(True)                        # its strides as given
        y = module.forward_act(xi, relu, residual)
        assert len(calls) == 1 and y.shape == x.shape
        y.backward(grad) if grad is not None else y.sum().backward()
        assert len(calls) == 2
    finally:
        BN.gather, BN.sync_group = old
    return y, xi.grad


ROUTES = ["fp16", "bf16", "frame-major", "channel-slice", "expanded-grad", "fp16-residual", "2-D", "3-D", "4-D", "momentum-None",
          "no-affine", "untracked"]


@pytest.mark.parametrize("route", ROUTES)
def test_module_route_is_the_contiguous_phases(route):
    c = 6
    shape = (5, c, 3, 7, 9) if route not in ("2-D", "3-D", "4-D") else {"2-D": (5, c), "3-D": (5, c, 40), "4-D": (5, c, 7, 9)}[route]
    sizes = [0, 2, 0, 3]
    g = torch.Generator().manual_seed(len(route))
    x = torch.randn(shape, generator=g).to(DEV) * 2 + 0.5
    dy = torch.ones(shape, device=DEV) if route == "expanded-grad" else torch.randn(shape, generator=g).to(DEV)
    res = torch.randn(shape, generator=g).to(DEV) if route == "fp16-residual" else None
    kw = {"momentum-None": dict(momentum=None), "no-affine": dict(affine=False), "untracked": dict(track_running_stats=False)}.get(route, {})
    dtype = {"fp16": torch.float16, "bf16": torch.bfloat16}.get(route, torch.float32)
    x = x.to(dtype)
    res = res.half() if res is not None else None
    def as5(t):                                                     # as the module reads it
        return t.reshape(0, c, 1, 1, 1) if t.numel() == 0 else t.reshape(t.shape[0], c, 1, 1, -1) if t.dim() != 5 else t
    xs, dys = torch.split(x, sizes), torch.split(dy, sizes)
    rs = torch.split(res, sizes) if res is not None else [None] * len(sizes)
    ref_mod = _module(c, **kw)
    gf, gb, ref = _phases([as5(t) for t in xs], ref_mod.weight, ref_mod.bias, [as5(t) if t is not None else None for t in rs],
                          [as5(t) for t in dys], True)
    for rank in range(len(sizes)):
        m = _module(c, **kw)
        xr = xs[rank]
        if route == "frame-major" and xr.numel():
            xr = TC.poisoned_frame_major(xr.float(), DEV)
        elif route == "channel-slice" and xr.numel():
            big = TC.poisoned(torch.cat([xr, xr[:, :3]], 1), DEV)
            xr = big[:, :c]
        grad = None if route == "expanded-grad" else dys[rank]
        y, gx = _drive(m, xr, rank, gf, gb, True, rs[rank], grad)
        yr, mean, var, count, dx, dw, db = ref[rank]
        assert torch.equal(y.reshape(yr.shape), yr), (route, rank)
        assert gx.dtype == xr.dtype and torch.equal(gx.reshape(dx.shape), dx.to(xr.dtype)), (route, rank)
        if m.affine:
            assert torch.equal(m.weight.grad, dw) and torch.equal(m.bias.grad, db), (route, rank)
        if m.track_running_stats:
            want = _module(c, **kw)
            BN.update_running_stats(want, mean, var, count)
            assert torch.equal(m.running_mean, want.running_mean) and torch.equal(m.running_var, want.running_var), (route, rank)
            assert int(m.num_batches_tracked) == 1
            # the group's count, not the rank's: torch's whole-batch update
            whole = nn.BatchNorm3d(c, **kw).to(DEV).double().train()
            whole(as5(x).double())
            assert torch.allclose(m.running_var.double(), whole.running_var, rtol=1e-5, atol=1e-6), (route, rank)


@pytest.mark.parametrize("shape", [(0, 8), (3, 8, 0), (2, 8, 0, 12), (2, 8, 3, 0, 5), (2, 8, 3, 4, 0), (0, 8, 3, 4, 5), (2, 8, 0, 4, 5)],
                         ids=_ids)
def test_an_input_with_no_elements_takes_part(shape):
    """a rank whose input has no elements, whichever dim is 0, takes part in one gather each way with n = 0 and moves its running
    statistics with the group's count"""
    other_x = torch.randn(3, 8, 6, 12, device=DEV) * 2 + 1
    other = BN.local_stats(f32_planes(other_x.reshape(3, 8, 1, 1, 72)))
    calls = []

    def gather(t, group):
        calls.append(t.clone())
        return torch.stack([t, other])
    old = BN.gather, BN.sync_group
    BN.gather, BN.sync_group = gather, (lambda norm: "group")
    try:
        norm = BN.FusedSyncBatchNorm(nn.SyncBatchNorm(8).to(DEV).train())
        x = torch.empty(shape, device=DEV, requires_grad=True)
        y = norm(x)
        assert y.shape == x.shape and len(calls) == 1
        assert bool((calls[0][:, 0] == 0).all())
        y.sum().backward()
        assert len(calls) == 2 and x.grad.shape == x.shape
    finally:
        BN.gather, BN.sync_group = old
    ref = nn.BatchNorm2d(8).to(DEV).double().train()
    ref(other_x.double())
    assert torch.allclose(norm.running_mean.double(), ref.running_mean, rtol=1e-5, atol=1e-6)
    assert torch.allclose(norm.running_var.double(), ref.running_var, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------------------------
# F: the SpatialGRU's step entries at worlds 2 to 4, every stage and gradient element by element
# ------------------------------------------------------------------------------------------------------------------------------
def _lockstep(ranks):
    results = [None] * len(ranks)
    triplets = [next(r) for r in ranks]
    while any(r is None for r in results):
        gathered = torch.stack(triplets)
        for i, r in enumerate(ranks):
            try:
                triplets[i] = r.send(gathered)
            except StopIteration as done:
                results[i] = done.value
    return results


GRU_CASES = [gc.CASES[i] for i in (0, 2, 3, 9, 12)] + [c for c in gc.CASES if c[7] != 0.0][:2] + \
    [c for c in gc.CASES if c[2] == 200 and c[3] == 200]                     # both 200 x 200 grids, one with bias_init 0.25
GRU_SPLITS = {2: lambda B: [0, B], 3: lambda B: [0, B - 1, 1], 4: lambda B: [0, 1, 0, B - 1]}


def abi_gru_group(x, h0, go, p, sizes, T, bias_init, need_h0=True):
    """The SpatialGRU's step entries for every rank of the batch split ``sizes``, the ranks in lockstep and a ``torch.stack`` of their
    triplets the gather, from NaN-poisoned inputs into guarded outputs: out, saved, means, vars, the step counts, each step's triplets,
    every gradient and both workspaces between sentinel margins, checked written and contained.  A rank with batch 0 (the step
    entries take batch >= 1) runs what the module runs for it: the batch norm's group entries on a (0, C_h, 1, X, Y) shape with NULL
    x / y / grad pointers.  Returns per rank (out, saved as (4, T, b, C_h, X, Y), means, vars, counts, grads dict)."""
    from fiery_b200 import future_prediction as FP
    lib = _lib.load()
    cx, ch, X, Y = x.shape[2], h0.shape[1], x.shape[3], x.shape[4]
    tx = x.shape[1]
    packed = FP.pack_weights([p["w_gates"][:ch], p["w_gates"][ch:], p["w_state"]], cx)
    bw, bb = p["gamma"], p["beta"]
    outs = _Outs()
    ranks = []
    for xr, hr, gr in zip(*(torch.split(t, sizes) for t in (x, h0, go))):
        b = xr.shape[0]
        r = dict(b=b, means=outs(T * ch, "means"), vars=outs(T * ch, "vars"), counts=outs(T, "counts", torch.float64))
        if b:
            xs, hs, gs = (TC.poisoned(t, DEV) for t in (xr, hr, gr))
            d = FP._desc(b, T, tx, X, Y, cx, ch, (xs.stride(0), xs.stride(1), xs.stride(2)), True, EPS, bias_init)
            r.update(d=d, x=xs, h0=hs, go=gs, out=outs(b * T * ch * X * Y, "out"), saved=outs(int(lib.fiery_spatial_gru_saved_bytes(d)) // 4, "saved"),
                     fws=outs(int(lib.fiery_spatial_gru_forward_workspace_bytes(d)) // 4, "forward workspace", must_write=False),
                     bws=outs(int(lib.fiery_spatial_gru_backward_workspace_bytes(d)) // 4, "backward workspace", must_write=False),
                     gx=outs(xr.numel(), "grad_x"), gh=outs(hr.numel(), "grad_h0", must_write=need_h0),
                     gwg=outs(p["w_gates"].numel(), "grad_w_gates"), gbg=outs(2 * ch, "grad_b_gates"),
                     gws=outs(p["w_state"].numel(), "grad_w_state"), gbw=outs(ch, "grad_bn_weight"), gbb=outs(ch, "grad_bn_bias"))
        else:
            d = _desc((0, ch, 1, X * Y), True, EPS)
            r.update(d=d, bnws=_workspace(d, outs, "empty rank's workspace"))
        ranks.append(r)
    ptr = lambda t: 0 if t is None else t.data_ptr()                              # noqa: E731
    for t in range(T):
        trip = []
        for r in ranks:
            st = outs(3 * ch, f"stats {t}", torch.float64)
            if r["b"]:
                _lib.call("fiery_spatial_gru_forward_step_begin", DEV, r["d"], t, r["x"].data_ptr(), r["h0"].data_ptr(), packed.data_ptr(),
                          p["b_gates"].data_ptr(), r["out"].data_ptr(), r["saved"].data_ptr(), st.data_ptr(), r["fws"].data_ptr())
            else:
                _lib.call("fiery_batch_norm_local_stats", DEV, r["d"], 0, st.data_ptr(), r["bnws"].data_ptr())
            trip.append(st.view(ch, 3))
        gathered = torch.stack(trip)
        for r in ranks:
            at = r["means"].data_ptr() + 4 * t * ch, r["vars"].data_ptr() + 4 * t * ch, r["counts"].data_ptr() + 8 * t
            if r["b"]:
                _lib.call("fiery_spatial_gru_forward_step_end", DEV, r["d"], t, len(ranks), gathered.data_ptr(), r["h0"].data_ptr(), ptr(bw),
                          ptr(bb), r["out"].data_ptr(), r["saved"].data_ptr(), r["means"].data_ptr(), r["vars"].data_ptr(), at[2],
                          r["fws"].data_ptr())
            else:
                _lib.call("fiery_batch_norm_forward_gathered", DEV, r["d"], len(ranks), gathered.data_ptr(), 0, ptr(bw), ptr(bb), 0, 0, *at,
                          r["bnws"].data_ptr())
    for t in reversed(range(T)):
        trip = []
        for r in ranks:
            sm = outs(3 * ch, f"sums {t}", torch.float64)
            if r["b"]:
                _lib.call("fiery_spatial_gru_backward_step_begin", DEV, r["d"], t, r["go"].data_ptr(), r["h0"].data_ptr(), r["out"].data_ptr(),
                          r["saved"].data_ptr(), r["means"].data_ptr(), r["vars"].data_ptr(), packed.data_ptr(), ptr(bw), ptr(bb),
                          r["gh"].data_ptr() if need_h0 else 0, sm.data_ptr(), r["bws"].data_ptr())
            else:
                at = r["means"].data_ptr() + 4 * t * ch, r["vars"].data_ptr() + 4 * t * ch
                _lib.call("fiery_batch_norm_local_grad_sums", DEV, r["d"], 0, 0, ptr(bw), ptr(bb), *at, sm.data_ptr(), 0, 0,
                          r["bnws"].data_ptr())
            trip.append(sm.view(ch, 3))
        gathered = torch.stack(trip)
        for r in ranks:
            if r["b"]:
                _lib.call("fiery_spatial_gru_backward_step_end", DEV, r["d"], t, len(ranks), gathered.data_ptr(), r["h0"].data_ptr(),
                          r["out"].data_ptr(), r["saved"].data_ptr(), r["means"].data_ptr(), r["vars"].data_ptr(), packed.data_ptr(), ptr(bw),
                          ptr(bb), r["gx"].data_ptr(), r["gh"].data_ptr() if need_h0 else 0, r["bws"].data_ptr())
            else:
                at = r["means"].data_ptr() + 4 * t * ch, r["vars"].data_ptr() + 4 * t * ch
                _lib.call("fiery_batch_norm_backward_gathered", DEV, r["d"], len(ranks), gathered.data_ptr(), 0, 0, ptr(bw), ptr(bb), *at, 0,
                          r["bnws"].data_ptr())
    for r in ranks:
        if r["b"]:
            _lib.call("fiery_spatial_gru_backward_weights", DEV, r["d"], r["x"].data_ptr(), r["h0"].data_ptr(), r["out"].data_ptr(),
                      r["saved"].data_ptr(), packed.data_ptr(), r["gwg"].data_ptr(), r["gbg"].data_ptr(), r["gws"].data_ptr(),
                      r["gbw"].data_ptr(), r["gbb"].data_ptr(), r["bws"].data_ptr())
    outs.check()
    if not need_h0:
        for r in ranks:
            if r["b"]:
                _untouched(r["gh"], "grad_h0")
    res = []
    for r in ranks:
        b = r["b"]
        if b:
            grads = {"x": r["gx"].view(b, tx, cx, X, Y), "h0": r["gh"].view(b, ch, X, Y) if need_h0 else None,
                     "w_gates": r["gwg"].view(p["w_gates"].shape), "b_gates": r["gbg"], "w_state": r["gws"].view(p["w_state"].shape),
                     "gamma": r["gbw"], "beta": r["gbb"]}
            res.append((r["out"].view(b, T, ch, X, Y), r["saved"][:4 * T * b * ch * X * Y].view(4, T, b, ch, X, Y),
                        r["means"].view(T, ch), r["vars"].view(T, ch), r["counts"], grads))
        else:
            res.append((None, None, r["means"].view(T, ch), r["vars"].view(T, ch), r["counts"], None))
    return res


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("case", GRU_CASES, ids=gc.case_id)
def test_spatial_gru_steps_against_fp64(case, world):
    """the step entries through the C ABI on guarded buffers, rank 0 empty (at world 3 without grad_h0, the carried gradient in the
    workspace): every stage and gradient of the whole batch element by element against the fp64 restatement, each within its bound;
    the same bits as the module's step generators"""
    from fiery_b200 import future_prediction as FP
    cx, ch, X, Y, b, T, Tx, bias_init = case
    B = b + 1
    p = gc.params(cx, ch, seed=cx + 3 * ch, dtype=torch.float32, device=DEV)
    x, h0, go = gc.inputs(B, T, Tx, cx, ch, X, Y, seed=world, dtype=torch.float32, device=DEV)
    sizes = GRU_SPLITS[world](B)
    need_h0 = world != 3
    got = abi_gru_group(x, h0, go, p, sizes, T, bias_init, need_h0)
    for _, _, m, v, n, _ in got:                                   # every rank's statistics and counts: the same bits
        assert torch.equal(m, got[0][2]) and torch.equal(v, got[0][3]) and torch.equal(n, got[0][4])
    assert bool((got[0][4] == B * X * Y).all())
    full = [g for g in got if g[0] is not None]
    out = torch.cat([g[0] for g in full])
    saved = torch.cat([g[1] for g in full], dim=2)
    stages, ref = gc.stage_ratios(gc.as_kernel(out, saved, got[0][2], got[0][3]), x, h0, p, T, True, EPS, bias_init)
    for k, (rr, _) in stages.items():
        _note(f"gru {k}", rr)
    bad = {k: v for k, v in stages.items() if not (v[1] and v[0] <= 1.0)}
    assert not bad, ("forward stages", bad)
    grads = {"x": torch.cat([g[5]["x"] for g in full]), "h0": torch.cat([g[5]["h0"] for g in full]) if need_h0 else None}
    for k in ("w_gates", "b_gates", "w_state", "gamma", "beta"):   # each rank's own: they add up to the whole batch's
        grads[k] = sum(g[5][k].double() for g in full)
    gr = gc.grad_ratios(ref, grads, x, h0, p, go, True, EPS)
    for k, (rr, _) in gr.items():
        _note(f"gru d_{k}", rr)
    bad = {k: v for k, v in gr.items() if not (v[1] and v[0] <= 1.0)}
    assert not bad, ("gradients", bad)
    # the module's generators drive the same entries: the same bits
    w_u, w_r, b_u, b_r = p["w_gates"][:ch], p["w_gates"][ch:], p["b_gates"][:ch], p["b_gates"][ch:]
    shards = [torch.split(t, sizes) for t in (x, h0, go)]
    fw = _lockstep([FP.sync_forward_steps(xr, hr, w_u, b_u, w_r, b_r, p["w_state"], p["gamma"], p["beta"], T, EPS, bias_init)
                    for xr, hr in zip(shards[0], shards[1])])
    bw = _lockstep([FP.sync_backward_steps(gr_, xr, hr, o, sv, m, v, w_u, w_r, p["w_state"], p["gamma"], p["beta"], T, EPS, bias_init,
                                           (True, need_h0) + (True,) * 7) for xr, hr, gr_, (o, m, v, _, sv) in zip(*shards, fw)])
    assert torch.equal(torch.cat([f[0] for f in fw]), out) and torch.equal(fw[0][1], got[0][2]) and torch.equal(fw[0][3], got[0][4])
    assert torch.equal(torch.cat([g[0] for g in bw]), grads["x"])
    for (o, m, v, n, sv), g in zip(fw, got):
        if g[0] is not None:
            assert torch.equal(sv.view(torch.float32)[:g[1].numel()], g[1].reshape(-1))
    for k, name in ((6, "w_state"), (7, "gamma"), (8, "beta")):
        for gb_, g in zip(bw, got):
            if g[0] is not None:
                assert torch.equal(gb_[k], g[5][name]), name


@pytest.mark.parametrize("exact", [False, True], ids=["random", "exact-regime"])
def test_spatial_gru_empty_rank_zero_is_the_operator(exact):
    """world 2 with rank 0 empty: every output and gradient bit for bit the through-time operator on rank 1's batch"""
    from fiery_b200 import future_prediction as FP
    if exact:
        x, h0, p, go = gc.exact_case(0, b=2, T=3)
        x, h0, go = (t.float().to(DEV) for t in (x, h0, go))
        p = {k: v.float().to(DEV) for k, v in p.items()}
        T, bias_init = 3, 0.0
    else:
        case = gc.CASES[3]
        cx, ch, X, Y, b, T, Tx, bias_init = case
        p = gc.params(cx, ch, seed=7, dtype=torch.float32, device=DEV)
        x, h0, go = gc.inputs(b, T, Tx, cx, ch, X, Y, seed=7, dtype=torch.float32, device=DEV)
    ch = h0.shape[1]
    w_u, w_r, b_u, b_r = p["w_gates"][:ch], p["w_gates"][ch:], p["b_gates"][:ch], p["b_gates"][ch:]
    args = (w_u, b_u, w_r, b_r, p["w_state"], p["gamma"], p["beta"])
    fw = _lockstep([FP.sync_forward_steps(t[:0] if k == 0 else t, hh[:0] if k == 0 else hh, *args, T, EPS, bias_init)
                    for k, (t, hh) in enumerate(((x, h0), (x, h0)))])
    need = (True,) * 9
    bw = _lockstep([FP.sync_backward_steps(go[:0] if k == 0 else go, x[:0] if k == 0 else x, h0[:0] if k == 0 else h0, o, sv, m, v, w_u, w_r,
                                           p["w_state"], p["gamma"], p["beta"], T, EPS, bias_init, need) for k, (o, m, v, _, sv) in enumerate(fw)])
    out, means, var, saved = FP.forward(x, h0, *args, None, None, T, True, EPS, bias_init)
    ref = FP.backward(go, x, h0, out, saved, means, var, w_u, w_r, p["w_state"], p["gamma"], p["beta"], T, True, EPS, bias_init, True, True,
                      True, True, True)
    o, m, v, n, sv = fw[1]
    assert torch.equal(o, out) and torch.equal(m, means) and torch.equal(v, var) and torch.equal(sv, saved)
    assert torch.equal(fw[0][1], means) and torch.equal(fw[0][2], var) and torch.equal(fw[0][3], n)
    for k, (a, e) in enumerate(zip(bw[1], ref)):
        assert torch.equal(a, e), k
    assert all(g is None or not bool(g.any()) for g in bw[0][2:])     # the empty rank's own parameter gradients are 0


# ------------------------------------------------------------------------------------------------------------------------------
# G: three processes on one GPU over gloo, rank 0 empty
# ------------------------------------------------------------------------------------------------------------------------------
G_BATCH = (0, 2, 1)


def _worker3(rank, world, port, q):
    from tests.test_sync_batch_norm_gpu import C, S, T_FUT, X, Y, _Holder
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        from fiery_b200 import install
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        ref = nn.SyncBatchNorm.convert_sync_batchnorm(_Holder()).to(dev).train()
        mine = copy.deepcopy(ref)
        install.use_fused_sync_batch_norm(mine)
        install.use_tensor_core_future_prediction(mine)
        g = torch.Generator().manual_seed(11)
        xs = [torch.randn(bb, S, C, X, Y, generator=g) for bb in G_BATCH]
        zs = [torch.randn(bb, T_FUT, 8, X, Y, generator=g) for bb in G_BATCH]
        hs = [torch.randn(bb, C, X, Y, generator=g) for bb in G_BATCH]
        x, z, h0 = xs[rank].to(dev), zs[rank].to(dev), hs[rank].to(dev)

        def run(m):
            xi, hi = x.clone().requires_grad_(True), h0.clone().requires_grad_(True)
            a, b = m(xi, z, hi)
            (a.sin().sum() + (b * b.detach().cos()).sum()).backward()
            grads = {}
            for n, p in m.named_parameters():                       # every rank reduces every parameter, in the same order
                v = p.grad.clone() if p.grad is not None else torch.zeros_like(p)
                dist.all_reduce(v)
                grads[n] = v / world
            return [a.detach(), b.detach(), xi.grad, hi.grad], grads, {n: bf.clone() for n, bf in m.named_buffers()}
        plain = [mm for mm in mine.modules() if type(mm) is nn.SyncBatchNorm]
        calls = {"gather": 0, "plain": 0}
        for mm in plain:
            mm.register_forward_hook(lambda *_: calls.__setitem__("plain", calls["plain"] + 1))
        o_ref, g_ref, s_ref = run(ref)
        real = {name: getattr(dist, name) for name in ("all_gather", "all_gather_into_tensor")}

        def counted(fn):
            def call(*a, **k):
                calls["gather"] += 1
                return fn(*a, **k)
            return call
        for name, fn in real.items():                   # the gradients' all_reduce inside run() is not counted
            setattr(dist, name, counted(fn))
        try:
            o, gr, st = run(mine)
        finally:
            for name, fn in real.items():
                setattr(dist, name, fn)
        # one gather per fused norm call each way, per GRU step each way (3 GRUs), and one per forward of torch's own norms: on the
        # empty rank too
        n_fused = sum(isinstance(mm, BN.FusedSyncBatchNorm) for mm in mine.temporal_model.modules())
        expected = 2 * n_fused + 2 * 3 * T_FUT + calls["plain"]
        host = lambda ts: [t.cpu().numpy() for t in ts]                                     # noqa: E731
        hostd = lambda d: {k: v.cpu().numpy() for k, v in d.items()}                        # noqa: E731
        q.put((rank, host(o), host(o_ref), hostd(gr), hostd(g_ref), hostd(st), hostd(s_ref), calls["gather"], expected))
    finally:
        dist.destroy_process_group()


def test_three_processes_over_gloo_with_rank_zero_empty():
    import tests.test_sync_batch_norm_gpu as S
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    world, port = len(G_BATCH), S._free_port()
    procs = [ctx.Process(target=_worker3, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = sorted([q.get(timeout=300) for _ in range(world)], key=lambda r: r[0])
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    dev = lambda x: [torch.from_numpy(a) for a in x] if isinstance(x, list) else {k: torch.from_numpy(a) for k, a in x.items()}  # noqa
    for r in res:
        assert r[7] == r[8] and r[7] > 0, ("gathers", r[0], r[7], r[8])
    res = [(r[0], *[dev(x) for x in r[1:7]]) for r in res]
    old = S.BATCH
    S.BATCH = G_BATCH
    try:
        o64s, g64, s64 = S._whole_batch_fp64()
        ot64s, gt64, st64 = S._whole_batch_fp64(tf32_gru_operands=True)
    finally:
        S.BATCH = old
    for rank, o, o_ref, gr, g_ref, st, s_ref in res:
        for i in range(4):
            if o64s[rank][i].numel():
                assert S._within(o[i], o_ref[i], o64s[rank][i], ot64s[rank][i]), (rank, i)
            else:
                assert o[i].numel() == 0
        for k in g_ref:
            assert S._within(gr[k], g_ref[k], g64[k], gt64[k]), (rank, k)
        for k in s_ref:
            if s_ref[k].is_floating_point():
                assert S._within(st[k], s_ref[k], s64[k], st64[k]), (rank, k)
            else:
                assert torch.equal(st[k], s_ref[k]), (rank, k)
    for _, _, _, _, _, st, _ in res[1:]:                             # the running statistics: bit for bit the same on every rank
        for k in res[0][5]:
            assert torch.equal(res[0][5][k], st[k]), k
