"""GPU: batch statistics over a process group on the batch-norm kernels (fiery_batch_norm_*_gathered, fiery_spatial_gru_*_step_*,
FusedSyncBatchNorm, the synced SpatialGRU).

* Simulated ranks in one process: a batch split into W uneven shards (a rank may hold none), each shard's local phase, a
  ``torch.stack`` standing in for the gather, then each shard's gathered phase -- against fp64 on the whole batch.  The batch norm
  runs tests/_batch_norm_cases.py's shapes; the SpatialGRU runs tests/_spatial_gru_cases.py's shapes through the per-step entries,
  the ranks' step generators driven in lockstep.
* World 1 through the phase entries is bit for bit the single-rank operators.
* Two processes on one GPU over gloo: a receptive-field-3 TemporalModel and a 3-GRU FuturePrediction converted with
  ``convert_sync_batchnorm``, swapped against torch's SyncBatchNorm, with the gathers counted.
"""
from __future__ import annotations

import copy
import datetime
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
import torch.nn.functional as F

from fiery_b200 import batch_norm as BN
from fiery_b200._lib import f32_planes
from tests import _batch_norm_cases as BNC
from tests import _spatial_gru_cases as GC

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 1e-5


def _rel(a, ref):
    return float((a.detach().double() - ref.detach().double()).norm() / ref.detach().double().norm().clamp_min(1e-30))


def _split(b, world):
    """uneven shard sizes of a batch of b over ``world`` ranks, weights 1 : 2 : 0 : 3 -- from W = 3 on one rank holds nothing"""
    weights = (1, 2, 0, 3)[:world]
    cuts = [round(b * sum(weights[:i]) / sum(weights)) for i in range(world + 1)]
    return [cuts[i + 1] - cuts[i] for i in range(world)]


def _reference(x, w, b, r, dy, relu):
    """fp64 whole-batch y and its gradients, and torch's fp32 CUDA error on y and dx"""
    def run(dtype):
        xi = x.to(dtype).requires_grad_(True)
        wi = w.to(dtype).requires_grad_(True) if w is not None else None
        bi = b.to(dtype).requires_grad_(True) if b is not None else None
        y = F.batch_norm(xi, None, None, wi, bi, True, 0.0, EPS)
        y = F.relu(y) if relu else y
        y = y + r.to(dtype) if r is not None else y
        y.backward(dy.to(dtype))
        return y.detach(), xi.grad, wi.grad if wi is not None else None, bi.grad if bi is not None else None
    return run(torch.float64), run(torch.float32)


def _simulated(shards, w, b, rs, dys, relu):
    xs = [f32_planes(s) for s in shards]
    gathered = torch.stack([BN.local_stats(x) for x in xs])
    fw = [BN.forward_gathered(gathered, x, w, b, r, EPS, relu) for x, r in zip(xs, rs)]
    sums = [BN.local_grad_sums(dy.contiguous(), x, w, b, f[1], f[2], EPS, relu, w is not None, b is not None)
            for x, dy, f in zip(xs, dys, fw)]
    gathered_b = torch.stack([s[0] for s in sums])
    dx = [BN.backward_gathered(gathered_b, dy.contiguous(), x, w, b, f[1], f[2], EPS, relu) for x, dy, f in zip(xs, dys, fw)]
    return fw, sums, dx


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("relu,residual,affine", [(True, True, True), (True, False, True), (False, False, True), (False, True, False)])
@pytest.mark.parametrize("shape", BNC.SHAPE_LIST, ids=lambda s: "x".join(map(str, s)))
def test_simulated_ranks_against_fp64(shape, relu, residual, affine, world):
    """tests/_batch_norm_cases.py's shapes split over simulated ranks, against fp64 on the whole batch; every rank's statistics, group
    count and running statistics bit for bit the same"""
    g = torch.Generator().manual_seed(sum(shape) + world)
    bsz, c = shape[0], shape[1]
    x = (torch.randn(shape, generator=g) * 2 + 0.5).to(DEV)
    dy = torch.randn(shape, generator=g).to(DEV)
    r = torch.randn(shape, generator=g).to(DEV) if residual else None
    w = (1 + 0.3 * torch.randn(c, generator=g)).to(DEV) if affine else None
    b = (0.3 * torch.randn(c, generator=g)).to(DEV) if affine else None
    sizes = _split(bsz, world)
    shards, dys = torch.split(x, sizes), torch.split(dy, sizes)
    rs = torch.split(r, sizes) if residual else [None] * world
    fw, sums, dx = _simulated(shards, w, b, rs, dys, relu)
    (y64, dx64, dw64, db64), (y32, dx32, _, _) = _reference(x, w, b, r, dy, relu)
    # every rank's statistics bit for bit the same
    for f in fw[1:]:
        for a, ref in zip(f[1:], fw[0][1:]):
            assert torch.equal(a, ref)
    assert float(fw[0][3]) == x.numel() // c
    # each rank moves its own running statistics with the group's count: bit for bit the same everywhere, torch's whole-batch update
    whole = nn.BatchNorm3d(c, momentum=0.25).to(DEV).double().train()
    whole(x.double())
    moved = []
    for _, mean, var, count in fw:
        bn = nn.BatchNorm3d(c, momentum=0.25).to(DEV).train()
        BN.update_running_stats(bn, mean, var, count)
        moved.append(bn)
    for bn in moved:
        assert torch.equal(bn.running_mean, moved[0].running_mean) and torch.equal(bn.running_var, moved[0].running_var)
        assert int(bn.num_batches_tracked) == 1
    assert torch.allclose(moved[0].running_mean.double(), whole.running_mean, rtol=1e-5, atol=1e-6)
    assert torch.allclose(moved[0].running_var.double(), whole.running_var, rtol=1e-5, atol=1e-6)
    y = torch.cat([f[0] for f in fw])
    assert _rel(y, y64) <= max(3 * _rel(y32, y64), 1e-6)
    # dx = scale (g' - S1 / n - x^ S2 / n) cancels to almost nothing when a channel has few values (2 in the 1-pixel shape): measure
    # its error against the size of the terms that cancel, scale g', when that is the larger
    terms = (dy.double() * (w.double().view(1, -1, 1, 1, 1) if affine else 1) / (x.double().var(dim=(0, 2, 3, 4), unbiased=False)
                                                                                  .view(1, -1, 1, 1, 1) + EPS).sqrt()).norm()
    size = max(float(dx64.norm()), float(terms))
    err, err_t = float((torch.cat(dx).double() - dx64).norm()) / size, float((dx32.double() - dx64).norm()) / size
    assert err <= max(3 * err_t, 1e-6), (err, err_t)
    mean64 = x.double().mean(dim=(0, 2, 3, 4))
    var64 = x.double().var(dim=(0, 2, 3, 4), unbiased=False)
    assert _rel(fw[0][1], mean64) < 1e-6 and _rel(fw[0][2], var64) < 1e-6
    if affine:
        # dgamma, dbeta per rank: that shard's own sums with the group's statistics; their sum the whole batch's gradient
        xh = (x.double() - mean64.view(1, -1, 1, 1, 1)) / (var64.view(1, -1, 1, 1, 1) + EPS).sqrt()
        pre = xh * w.double().view(1, -1, 1, 1, 1) + b.double().view(1, -1, 1, 1, 1)
        gm = dy.double() * (pre > 0) if relu else dy.double()
        for (_, dw_r, db_r), gs, xs in zip(sums, torch.split(gm, sizes), torch.split(xh, sizes)):
            assert torch.allclose(db_r.double(), gs.sum(dim=(0, 2, 3, 4)), rtol=1e-4, atol=1e-4 * gm.abs().sum() / c)
            assert torch.allclose(dw_r.double(), (gs * xs).sum(dim=(0, 2, 3, 4)), rtol=1e-4, atol=1e-4 * gm.abs().sum() / c)
        assert _rel(sum(s[1] for s in sums), dw64) < 1e-4 and _rel(sum(s[2] for s in sums), db64) < 1e-4


@pytest.mark.parametrize("relu,residual", [(True, True), (False, False)])
def test_world_one_is_batch_norm_act_bit_for_bit(relu, residual):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 35, 2, 33, 130, generator=g).to(DEV)
    dy = torch.randn(x.shape, generator=g).to(DEV)
    r = torch.randn(x.shape, generator=g).to(DEV) if residual else None
    w, b = (1 + 0.3 * torch.randn(35, generator=g)).to(DEV), (0.3 * torch.randn(35, generator=g)).to(DEV)
    y0, m0, v0 = torch.ops.fiery_b200.batch_norm_act(x, w, b, None, None, r, True, EPS, relu)
    dx0, dw0, db0 = torch.ops.fiery_b200.batch_norm_act_backward(dy, x, w, b, m0, v0, True, EPS, relu, True, True, True)
    fw, sums, dx = _simulated([x], w, b, [r], [dy], relu)
    y, m, v, n = fw[0]
    assert torch.equal(y, y0) and torch.equal(m, m0) and torch.equal(v, v0) and float(n) == x.numel() // 35
    assert torch.equal(dx[0], dx0) and torch.equal(sums[0][1], dw0) and torch.equal(sums[0][2], db0)


def test_world_one_running_statistics_match_the_fused_module():
    """a FusedSyncBatchNorm's synced Function at world 1 moves the running statistics as FusedBatchNorm3d does"""
    bn = nn.BatchNorm3d(16).to(DEV)
    ref = BN.FusedBatchNorm3d(copy.deepcopy(bn))
    mine = BN.FusedSyncBatchNorm(nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(bn)))
    x = torch.randn(2, 16, 3, 8, 12, device=DEV)
    y0 = ref.forward_act(x, relu=True)
    y, mean, var, count = BN.SyncBatchNormAct.apply(x, mine.weight, mine.bias, None, EPS, True, lambda t: t[None])
    mine.update_running_stats(mean, var, count)
    assert torch.equal(y, y0)
    assert torch.equal(mine.running_mean, ref.running_mean) and torch.equal(mine.running_var, ref.running_var)
    assert int(mine.num_batches_tracked) == int(ref.num_batches_tracked) == 1


def test_an_empty_rank_takes_part(monkeypatch):
    """a rank whose 4-D input is empty (the norm of an unswapped SpatialGRU) still gathers, and moves its running statistics with the
    other rank's: here the group is this empty rank and a rank holding x"""
    x = torch.randn(3, 8, 6, 12, device=DEV) * 2 + 1
    other = BN.local_stats(f32_planes(x.reshape(3, 8, 1, 1, 72)))
    calls = []
    monkeypatch.setattr(BN, "sync_group", lambda norm: "group")
    monkeypatch.setattr(BN, "gather", lambda t, group: calls.append(group) or torch.stack([t, other]))
    norm = BN.FusedSyncBatchNorm(nn.SyncBatchNorm(8).to(DEV).train())
    y = norm(torch.empty(0, 8, 6, 12, device=DEV, requires_grad=True))
    assert y.shape == (0, 8, 6, 12) and calls == ["group"]
    ref = nn.BatchNorm2d(8).to(DEV).double().train()
    ref(x.double())
    assert torch.allclose(norm.running_mean.double(), ref.running_mean, rtol=1e-5, atol=1e-6)
    assert torch.allclose(norm.running_var.double(), ref.running_var, rtol=1e-5, atol=1e-6)
    y.sum().backward()
    assert calls == ["group", "group"]


def test_spatial_gru_world_one_is_the_operator_bit_for_bit():
    from fiery_b200.future_prediction import SyncSpatialGRU
    from oracle.future_oracle import SpatialGRU
    g = torch.Generator().manual_seed(5)
    base = SpatialGRU(24, 40).to(DEV)
    with torch.no_grad():
        for p in base.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if p.dim() == 1 and p.shape[0] == 40 else 0.0))
    b, T, h, w = 2, 4, 12, 16
    x = torch.randn(b, T, 24, h, w, generator=g).to(DEV)
    h0 = torch.randn(b, 40, h, w, generator=g).to(DEV)
    go = torch.randn(b, T, 40, h, w, generator=g).to(DEV)
    params = [base.conv_update.weight, base.conv_update.bias, base.conv_reset.weight, base.conv_reset.bias,
              base.conv_state_tilde.conv.weight, base.conv_state_tilde.norm.weight, base.conv_state_tilde.norm.bias]

    def run(fn):
        xi, hi = x.clone().requires_grad_(True), h0.clone().requires_grad_(True)
        for p in params:
            p.grad = None
        out, means, var = fn(xi, hi)[:3]
        out.backward(go)
        return [out, means, var, xi.grad, hi.grad] + [p.grad.clone() for p in params]
    ref = run(lambda xi, hi: torch.ops.fiery_b200.spatial_gru(xi, hi, *params, None, None, T, True, EPS, 0.0))
    got = run(lambda xi, hi: SyncSpatialGRU.apply(xi, hi, *params, T, EPS, 0.0, lambda t: t[None]))
    for i, (a, r) in enumerate(zip(got, ref)):
        assert torch.equal(a, r), i


# ------------------------------------------------------------------------------------------------------------------------------
# the SpatialGRU's per-step entries, simulated ranks in lockstep
# ------------------------------------------------------------------------------------------------------------------------------
def _lockstep(ranks):
    """run the ranks' step generators (future_prediction.sync_*_steps) together, a torch.stack of their triplets standing in for the
    gather at every step; returns each rank's result"""
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


GRU_SPLITS = {1: lambda b: [b + 1], 2: lambda b: [1, b], 3: lambda b: [b, 0, 1]}     # a batch of b + 1, uneven; W = 3: an empty rank
_GRU_REFERENCES = {}


def _gru_case(i):
    """(module, inputs, variant) of _spatial_gru_cases.CASES[i]: every third case without the norm's affine parameters, every other one
    without grad_h0 (the carried gradient then lives in the workspace)"""
    from oracle.future_oracle import SpatialGRU
    from tests.test_spatial_gru_gpu import _randomize
    cx, ch, X, Y, b, T, Tx, bias_init = GC.CASES[i]
    affine, need_h0 = i % 3 != 1, i % 2 == 0
    base = _randomize(SpatialGRU(cx, ch, gru_bias_init=bias_init), 100 + i).to(DEV).train()
    if not affine:                                                 # running statistics drawn as _randomize draws them
        norm = nn.BatchNorm2d(ch, affine=False)
        g = torch.Generator().manual_seed(200 + i)
        norm.running_mean.copy_(torch.randn(ch, generator=g) * 0.1)
        norm.running_var.copy_(torch.rand(ch, generator=g) + 0.5)
        base.conv_state_tilde.norm = norm.to(DEV).train()
    g = torch.Generator().manual_seed(i)
    B = b + 1
    x = torch.randn(B, Tx, cx, X, Y, generator=g).to(DEV)
    h0 = torch.randn(B, ch, X, Y, generator=g).to(DEV)
    gout = torch.randn(B, T, ch, X, Y, generator=g).to(DEV)
    return base, (x, h0, gout), (affine, need_h0, T, bias_init)


def _gru_params(m):
    n = m.conv_state_tilde.norm
    return (m.conv_update.weight, m.conv_update.bias, m.conv_reset.weight, m.conv_reset.bias, m.conv_state_tilde.conv.weight, n.weight,
            n.bias)


def _gru_reference(i, base, x, h0, gout, T):
    """the oracle module on the whole batch: fp64, torch's fp32 and fp64 on TF32-rounded operands (the GRU tests' bar)"""
    if i not in _GRU_REFERENCES:
        from tests.test_spatial_gru_gpu import _tf32_operands

        def run(m, dtype):
            xi = x.detach().to(dtype, copy=True).requires_grad_(True)
            hi = h0.detach().to(dtype, copy=True).requires_grad_(True)
            out = m(xi.expand(-1, T, -1, -1, -1), hi)
            out.backward(gout.to(dtype))
            grads = {"out": out.detach(), "x": xi.grad, "h0": hi.grad}
            grads.update({n: p.grad for n, p in m.named_parameters()})
            norm = m.conv_state_tilde.norm
            return grads, (norm.running_mean.clone(), norm.running_var.clone(), int(norm.num_batches_tracked))
        _GRU_REFERENCES.clear()                                     # one case at a time: the 200 x 200 ones are large
        _GRU_REFERENCES[i] = (run(copy.deepcopy(base).double(), torch.float64), run(copy.deepcopy(base), torch.float32),
                              run(_tf32_operands(copy.deepcopy(base).double()), torch.float64))
    return _GRU_REFERENCES[i]


@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("i", range(len(GC.CASES)), ids=[GC.case_id(c) for c in GC.CASES])
def test_spatial_gru_simulated_ranks(i, world):
    """tests/_spatial_gru_cases.py's shapes through fiery_spatial_gru_*_step_*, each rank with its own saved buffer and workspace:
    world 1 bit for bit the through-time operator, worlds 2 and 3 against the fp64 oracle module on the whole batch within the GRU
    tests' bar, and every rank's running statistics after T steps the same bits"""
    from fiery_b200 import future_prediction as FP
    from tests.test_spatial_gru_gpu import _within
    base, (x, h0, gout), (affine, need_h0, T, bias_init) = _gru_case(i)
    w_u, b_u, w_r, b_r, w_s, bn_w, bn_b = (p.detach() if p is not None else None for p in _gru_params(base))
    need = (True, need_h0, True, True, True, True, True, affine, affine)
    sizes = GRU_SPLITS[world](x.shape[0] - 1)
    shards = [torch.split(t, sizes) for t in (x, h0, gout)]
    fw = _lockstep([FP.sync_forward_steps(xr, hr, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b, T, EPS, bias_init)
                    for xr, hr in zip(shards[0], shards[1])])
    bw = _lockstep([FP.sync_backward_steps(gr, xr, hr, o, sv, m, v, w_u, w_r, w_s, bn_w, bn_b, T, EPS, bias_init, need)
                    for xr, hr, gr, (o, m, v, _, sv) in zip(*shards, fw)])
    for o, m, v, n, _ in fw[1:]:                                   # every rank's statistics and counts: the same bits
        assert torch.equal(m, fw[0][1]) and torch.equal(v, fw[0][2]) and torch.equal(n, fw[0][3])
    assert torch.equal(fw[0][3], torch.full((T,), float(x.shape[0] * x.shape[3] * x.shape[4]), dtype=torch.float64, device=DEV))
    moved = []
    for _, m, v, n, _ in fw:
        norm = copy.deepcopy(base.conv_state_tilde.norm)
        for t in range(T):
            BN.update_running_stats(norm, m[t], v[t], n[t:t + 1])
        moved.append(norm)
    for norm in moved:
        assert torch.equal(norm.running_mean, moved[0].running_mean) and torch.equal(norm.running_var, moved[0].running_var)
        assert int(norm.num_batches_tracked) == T
    if world == 1:
        out, means, var, saved = FP.forward(x, h0, w_u, b_u, w_r, b_r, w_s, bn_w, bn_b, None, None, T, True, EPS, bias_init)
        ref = FP.backward(gout, x, h0, out, saved, means, var, w_u, w_r, w_s, bn_w, bn_b, T, True, EPS, bias_init, True, need_h0, True,
                          True, affine)
        o, m, v, _, sv = fw[0]
        assert torch.equal(o, out) and torch.equal(m, means) and torch.equal(v, var) and torch.equal(sv, saved)
        for k, (a, r) in enumerate(zip(bw[0], ref)):
            assert (a is None) == (r is None), k
            assert a is None or torch.equal(a, r), k
        return
    (g64, s64), (g32, s32), (gt, st) = _gru_reference(i, base, x, h0, gout, T)
    got = {"out": torch.cat([f[0] for f in fw]), "x": torch.cat([g[0] for g in bw])}
    if need_h0:
        got["h0"] = torch.cat([g[1] for g in bw])
    names = ["conv_update.weight", "conv_update.bias", "conv_reset.weight", "conv_reset.bias", "conv_state_tilde.conv.weight"]
    names += ["conv_state_tilde.norm.weight", "conv_state_tilde.norm.bias"] if affine else []
    for k, name in enumerate(names):                               # each rank's parameter gradient is its own: they add up
        got[name] = sum(g[2 + k] for g in bw)
    for k, a in got.items():
        e, e_ref = _rel(a, g64[k]), max(_rel(g32[k], g64[k]), _rel(gt[k], g64[k]))
        assert _within(e, e_ref), (k, e, e_ref)
    assert int(s64[2]) == T
    for k, a in enumerate((moved[0].running_mean, moved[0].running_var)):    # the same bar: a mean near 0 carries s's TF32 rounding
        e, e_ref = _rel(a, s64[k]), max(_rel(s32[k], s64[k]), _rel(st[k], s64[k]))
        assert _within(e, e_ref), (("running_mean", "running_var")[k], e, e_ref)


# ------------------------------------------------------------------------------------------------------------------------------
# two processes on one GPU over gloo
# ------------------------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


C, X, Y, S, T_FUT = 16, 12, 16, 3, 3
BATCH = (2, 1)                                               # per-rank batch: uneven


class _Holder(nn.Module):
    def __init__(self):
        super().__init__()
        from oracle.future_oracle import FuturePrediction
        from oracle.temporal_oracle import TemporalModel
        torch.manual_seed(0)
        self.temporal_model = TemporalModel(C, 3, (X, Y), start_out_channels=C)
        self.future_prediction = FuturePrediction(C, 8, n_gru_blocks=3, n_res_layers=1)

    def forward(self, x, z, h0):
        return self.temporal_model(x), self.future_prediction(z, h0)


def _worker(rank, world, port, backend, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        from fiery_b200 import install
        dev = torch.device("cuda", rank % torch.cuda.device_count())
        torch.cuda.set_device(dev)
        ref = nn.SyncBatchNorm.convert_sync_batchnorm(_Holder()).to(dev).train()
        mine = copy.deepcopy(ref)
        install.use_fused_sync_batch_norm(mine)
        install.use_tensor_core_future_prediction(mine)
        g = torch.Generator().manual_seed(11)
        xs = [torch.randn(bb, S, C, X, Y, generator=g) for bb in BATCH]
        zs = [torch.randn(bb, T_FUT, 8, X, Y, generator=g) for bb in BATCH]
        hs = [torch.randn(bb, C, X, Y, generator=g) for bb in BATCH]
        x, z, h0 = xs[rank].to(dev), zs[rank].to(dev), hs[rank].to(dev)

        def run(m, dtype=torch.float32):
            xi, hi = x.to(dtype, copy=True).requires_grad_(True), h0.to(dtype, copy=True).requires_grad_(True)
            a, b = m(xi, z.to(dtype), hi)
            (a.sin().sum() + (b * b.detach().cos()).sum()).backward()
            grads = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
            for v in grads.values():
                dist.all_reduce(v)
                v /= world
            stats = {n: bf.clone() for n, bf in m.named_buffers()}
            return [a.detach(), b.detach(), xi.grad, hi.grad], grads, stats

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
        for name, fn in real.items():                   # gloo gathers with all_gather, NCCL with all_gather_into_tensor
            setattr(dist, name, counted(fn))
        try:
            o, gr, st = run(mine)
        finally:
            for name, fn in real.items():
                setattr(dist, name, fn)
        n_fused = sum(isinstance(mm, BN.FusedSyncBatchNorm) for mm in mine.temporal_model.modules())
        expected = 2 * n_fused + 2 * 3 * T_FUT + calls["plain"]
        # numpy arrays: plain pickles that outlive the worker (a shared tensor's storage would not)
        host = lambda ts: [t.cpu().numpy() for t in ts]                                     # noqa: E731
        hostd = lambda d: {k: v.cpu().numpy() for k, v in d.items()}                        # noqa: E731
        q.put((rank, host(o), host(o_ref), hostd(gr), hostd(g_ref), hostd(st), hostd(s_ref), calls["gather"], expected))
    finally:
        dist.destroy_process_group()


def _spawn(backend):
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = sorted([q.get(timeout=300) for _ in range(world)], key=lambda r: r[0])
        dev = lambda x: [torch.from_numpy(a) for a in x] if isinstance(x, list) else {k: torch.from_numpy(a) for k, a in x.items()}  # noqa
        res = [(r[0], *[dev(x) for x in r[1:7]], r[7], r[8]) for r in res]
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    return res


def _within(got, ref32, ref64, tf64):
    """the GRU tests' bar: 3x the larger of torch's own fp32 error and fp64 on TF32-rounded operands, against fp64, and never below
    1e-3 (the TF32 operand rounding)"""
    return _rel(got, ref64) <= max(3 * max(_rel(ref32, ref64), _rel(tf64, ref64)), 1e-3)


def _whole_batch_fp64(tf32_gru_operands=False):
    """the group's computation in one process: the same model with plain BatchNorms, in fp64, on the ranks' shards concatenated
    (with ``tf32_gru_operands`` the GRUs' convolutions take TF32-rounded operands, as the kernels do).  Returns each rank's slice of
    the outputs and input gradients, the parameter gradients over the ranks' mean loss, and the running statistics."""
    from tests.test_spatial_gru_gpu import _tf32_operands
    m = _Holder().cuda().double().train()
    if tf32_gru_operands:
        _tf32_operands(m.future_prediction.spatial_grus)
    g = torch.Generator().manual_seed(11)
    xs = [torch.randn(bb, S, C, X, Y, generator=g) for bb in BATCH]
    zs = [torch.randn(bb, T_FUT, 8, X, Y, generator=g) for bb in BATCH]
    hs = [torch.randn(bb, C, X, Y, generator=g) for bb in BATCH]
    x, z, h0 = (torch.cat(t).cuda().double() for t in (xs, zs, hs))
    x.requires_grad_(True)
    h0.requires_grad_(True)
    a, b = m(x, z, h0)
    (a.sin().sum() + (b * b.detach().cos()).sum()).backward()
    grads = {n: p.grad.cpu() / len(BATCH) for n, p in m.named_parameters()}
    stats = {n: bf.cpu() for n, bf in m.named_buffers()}
    cuts = [0] + list(torch.tensor(BATCH).cumsum(0))
    per_rank = [[t.detach().cpu()[cuts[r]:cuts[r + 1]] for t in (a, b, x.grad, h0.grad)] for r in range(len(BATCH))]
    return per_rank, grads, stats


def _check(res):
    o64s, g64, s64 = _whole_batch_fp64()
    ot64s, gt64, st64 = _whole_batch_fp64(tf32_gru_operands=True)
    for rank, o, o_ref, gr, g_ref, st, s_ref, n_gather, expected in res:
        o64, ot64 = o64s[rank], ot64s[rank]
        assert n_gather == expected, (rank, n_gather, expected)
        for i in range(4):
            assert _within(o[i], o_ref[i], o64[i], ot64[i]), (rank, i, _rel(o[i], o64[i]), _rel(o_ref[i], o64[i]), _rel(ot64[i], o64[i]))
        for k in g_ref:
            assert _within(gr[k], g_ref[k], g64[k], gt64[k]), (rank, k, _rel(gr[k], g64[k]), _rel(g_ref[k], g64[k]), _rel(gt64[k], g64[k]))
        for k in s_ref:
            if s_ref[k].is_floating_point():
                assert _within(st[k], s_ref[k], s64[k], st64[k]), k
            else:
                assert torch.equal(st[k], s_ref[k]), k
    # the running statistics: bit for bit the same on both ranks
    for k in res[0][5]:
        assert torch.equal(res[0][5][k], res[1][5][k]), k


def test_two_processes_over_gloo():
    _check(_spawn("gloo"))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL needs one GPU per rank")
def test_two_processes_over_nccl():
    _check(_spawn("nccl"))
