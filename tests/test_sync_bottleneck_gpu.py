"""GPU: the future prediction's Bottleneck with its norms' statistics over a process group (fiery_bottleneck_sync_*_stage,
bottleneck.sync_*_stages, SyncBottleneck, TensorCoreBottleneck over FusedSyncBatchNorm norms).

* World 1 is the single-rank C ABI bit for bit over tests/_bottleneck_cases.py's shapes.
* Simulated ranks in one process, their stage generators driven in lockstep with a ``torch.stack`` standing in for the gather: each
  rank bit for bit the chain of the existing group entry points (fiery_batch_norm_local_stats / _forward_gathered / _local_grad_sums /
  _backward_gathered between the entry and 3x3 kernels), the statistics, counts and running statistics the same bits on every rank,
  and the whole batch against an fp64 oracle Bottleneck.
* Each gradient alone, the scale-0 / shift-1 padding, autocast, and eval / world 1 through the module.
* Two processes on one GPU over gloo (and NCCL with two GPUs): a converted FuturePrediction with every swap against torch's
  SyncBatchNorm model, the gathers counted.
"""
from __future__ import annotations

import copy
import datetime
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from fiery_b200 import _lib
from fiery_b200 import batch_norm as BN
from fiery_b200 import bottleneck as bk
from oracle.future_oracle import Bottleneck, FuturePrediction
from tests._bottleneck_cases import (GRAD_KEYS, SHAPES, _call, _conv_desc, _entry_desc, _entry_dgrad, _entry_fwd, _entry_pack,
                                     _entry_wgrad, fused_backward, fused_forward, margins_intact, nan_filled, operands)
from tests.test_sync_batch_norm_gpu import _free_port

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 1e-5


def _ids(s):
    return "x".join(str(v) for v in s)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _rel(a, ref):
    return float((a.detach().double() - ref.detach().double()).norm() / ref.detach().double().norm().clamp_min(1e-30))


def _affine(norms):
    """the 6 weights and biases of operands()' 12 norm parameters"""
    return [norms[i] for i in (0, 1, 4, 5, 8, 9)]


def _lockstep(ranks):
    """run the ranks' stage generators together, a torch.stack of their triplets standing in for each gather (every rank gathers as
    often, possibly never); returns each rank's result"""
    results, triplets, gathered = [None] * len(ranks), [None] * len(ranks), None
    while True:
        for i, r in enumerate(ranks):
            try:
                triplets[i] = next(r) if gathered is None else r.send(gathered)
            except StopIteration as done:
                results[i], triplets[i] = done.value, None
        if all(t is None for t in triplets):
            return results
        gathered = torch.stack(triplets)


def _counting(gen, calls):
    """gen, with each triplet it yields appended to ``calls``"""
    try:
        t = next(gen)
        while True:
            calls.append(t)
            t = gen.send((yield t))
    except StopIteration as done:
        return done.value


def _sync(shards, gouts, weights, params, need=(True,) * 10):
    """each rank's (forward, gradients) through the stage generators in lockstep"""
    fw = _lockstep([bk.sync_forward_stages(x, *weights, params, EPS) for x in shards])
    bw = _lockstep([bk.sync_backward_stages(g, x, *f[1:5], *weights, params, EPS, list(need)) for x, g, f in zip(shards, gouts, fw)])
    return fw, bw


@pytest.mark.parametrize("shape", SHAPES, ids=_ids)
def test_a_group_of_one_is_the_single_rank_path_bit_for_bit(shape):
    x, weights, norms = operands(*shape, seed=sum(shape))
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    (out, y1, y2, y3, stats), _ = fused_forward(x, weights, norms, True)
    grads, _ = fused_backward(g, x, y1, y2, y3, stats, weights, norms, True)
    (fw,), (bw,) = _sync([x], [g], weights, _affine(norms))
    for name, got, ref in zip(("out", "y1", "y2", "y3", "stats"), fw, (out, y1, y2, y3, stats)):
        assert _bits_equal(got, ref), name
    assert torch.equal(fw[5], torch.full((3,), float(shape[0] * shape[2] * shape[3]), dtype=torch.float64, device=DEV))
    for name, got, ref in zip(GRAD_KEYS, bw, grads):
        assert _bits_equal(got, ref), name


# ------------------------------------------------------------------------------------------------------------------------------
# simulated ranks against the chain of the existing group entry points
# ------------------------------------------------------------------------------------------------------------------------------
def _5d(t):
    return t.view(t.shape[0], t.shape[1], 1, t.shape[2], t.shape[3])


def _chain_forward(x, weights, params):
    """one rank's forward as the existing entry points compute it, yielding each norm's local triplet: dict of y1, y2, y3, a1, a2,
    out, stats and counts"""
    maps, c, h, w = x.shape
    m, p = c // 2, h * w
    w_d, w_c, w_u = weights
    r = {"stats": [], "counts": []}

    def norm(i, y, residual=None):
        gathered = yield BN.local_stats(_5d(y))
        a, mean, var, count = BN.forward_gathered(gathered, _5d(y), params[2 * i], params[2 * i + 1], residual, EPS, True)
        r["stats"] += [mean, var]
        r["counts"].append(count)
        return a.view(y.shape)
    if maps == 0:
        for i, k in enumerate((m, m, c)):
            yield from norm(i, x.new_empty((0, k, h, w)))
        return r
    dd, du, cd = _entry_desc(maps, c, m, p), _entry_desc(maps, m, c, p), _conv_desc(maps, m, h, w)
    pd, pu = _entry_pack(dd, w_d.reshape(m, c)), _entry_pack(du, w_u.reshape(c, m))
    pc = torch.empty(int(_lib.load().fiery_causal_conv3d_packed_bytes(cd)), dtype=torch.uint8, device=x.device)
    _call("fiery_causal_conv3d_pack_weights", x.device, cd, w_c.contiguous().data_ptr(), pc.data_ptr())
    r.update(dd=dd, du=du, cd=cd, pd=pd, pu=pu, pc=pc)
    r["y1"] = _entry_fwd(dd, x, pd, m)
    r["a1"] = yield from norm(0, r["y1"])
    r["y2"] = torch.empty_like(r["y1"])
    _call("fiery_causal_conv3d_forward", x.device, cd, r["a1"].data_ptr(), pc.data_ptr(), r["y2"].data_ptr())
    r["a2"] = yield from norm(1, r["y2"])
    r["y3"] = _entry_fwd(du, r["a2"], pu, c)
    r["out"] = yield from norm(2, r["y3"], _5d(x))
    return r


def _chain_backward(g, x, weights, params, f):
    """the gradients as the existing entry points compute them from ``_chain_forward``'s f, yielding each norm's local sums"""
    maps, c, h, w = x.shape
    m = c // 2
    means, vars_ = f["stats"][0::2], f["stats"][1::2]
    r = {}

    def norm(i, y, dy):
        sums, r[f"gw{i + 1}"], r[f"gb{i + 1}"] = BN.local_grad_sums(_5d(dy), _5d(y), params[2 * i], params[2 * i + 1], means[i], vars_[i],
                                                                    EPS, True, True, True)
        gathered = yield sums
        if maps:
            return BN.backward_gathered(gathered, _5d(dy), _5d(y), params[2 * i], params[2 * i + 1], means[i], vars_[i], EPS,
                                        True).view(y.shape)
    if maps == 0:
        for i, k in ((2, c), (1, m), (0, m)):
            yield from norm(i, x.new_empty((0, k, h, w)), x.new_empty((0, k, h, w)))
        return r
    dy3 = yield from norm(2, f["y3"], g)
    r["gW_up"] = _entry_wgrad(f["du"], f["a2"], dy3, c, m).view(c, m, 1, 1)
    da2 = _entry_dgrad(f["du"], dy3, f["pu"], m)
    dy2 = yield from norm(1, f["y2"], da2)
    r["gW_conv"] = torch.empty_like(weights[1])
    ws = _lib.workspace(_lib.load().fiery_causal_conv3d_backward_weight_workspace_bytes(f["cd"]), x.device)
    _call("fiery_causal_conv3d_backward_weight", x.device, f["cd"], f["a1"].data_ptr(), dy2.data_ptr(), r["gW_conv"].data_ptr(),
          ws.data_ptr())
    da1 = torch.empty_like(dy2)
    _call("fiery_causal_conv3d_backward_data", x.device, f["cd"], dy2.data_ptr(), f["pc"].data_ptr(), da1.data_ptr())
    dy1 = yield from norm(0, f["y1"], da1)
    r["gW_down"] = _entry_wgrad(f["dd"], x, dy1, m, c).view(m, c, 1, 1)
    r["dx"] = _entry_dgrad(f["dd"], dy1, f["pd"], c) + g
    return r


SPLITS = {2: (1, 2), 3: (1, 0, 2), 4: (1, 2, 0, 3)}           # uneven; from W = 3 on one rank holds nothing


def _split(n, world):
    weights = SPLITS[world]
    cuts = [round(n * sum(weights[:i]) / sum(weights)) for i in range(world + 1)]
    return [cuts[i + 1] - cuts[i] for i in range(world)]


def _oracle(c, weights, params):
    """the oracle Bottleneck holding these weights and norm parameters, momentum 0.1"""
    b = Bottleneck(c)
    norms = [b.layers.abn_down_project[0], b.layers.abn[0], b.layers.abn_up_project[0]]
    with torch.no_grad():
        for conv, wt in zip((b.layers.conv_down_project, b.layers.conv, b.layers.conv_up_project), weights):
            conv.weight.copy_(wt)
        for i, bn in enumerate(norms):
            bn.weight.copy_(params[2 * i])
            bn.bias.copy_(params[2 * i + 1])
            bn.momentum = 0.1
    return b.to(DEV).train()


def _oracle_step(block, x, g, dtype):
    block = copy.deepcopy(block).to(dtype)
    xi = x.to(dtype).requires_grad_(True)
    out = block(xi)
    out.backward(g.to(dtype))
    grads = [xi.grad] + [p.grad for p in block.parameters()]
    return [out.detach()] + grads, block


# (shape, world): the shapes of tests/_bottleneck_cases.py small enough to run three times with their fp64 references
GROUP_CASES = [(s, wd) for s in [(12, 64, 200, 200), (12, 70, 33, 20), (3, 64, 9, 36), (2, 17, 8, 16)] for wd in (2, 3, 4)]


@pytest.mark.parametrize("shape,world", GROUP_CASES, ids=[f"{_ids(s)}-w{wd}" for s, wd in GROUP_CASES])
def test_simulated_ranks(shape, world):
    maps, c, h, w = shape
    x, weights, norms = operands(*shape, seed=sum(shape) + world)
    params = _affine(norms)
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(world)).to(DEV)
    sizes = _split(maps, world)
    assert world < 3 or 0 in sizes
    shards, gouts = torch.split(x, sizes), torch.split(g, sizes)
    fw, bw = _sync(shards, gouts, weights, params)
    chain_f = _lockstep([_chain_forward(xr, weights, params) for xr in shards])
    chain_b = _lockstep([_chain_backward(gr, xr, weights, params, f) for xr, gr, f in zip(shards, gouts, chain_f)])
    # each rank: the chain of the existing group entry points, bit for bit
    for r, (f, b, cf, cb) in enumerate(zip(fw, bw, chain_f, chain_b)):
        assert _bits_equal(f[4], torch.cat(cf["stats"])), r
        assert torch.equal(f[5], torch.cat(cf["counts"])), r
        if sizes[r]:
            for name, got in zip(("out", "y1", "y2", "y3"), f[:4]):
                assert _bits_equal(got, cf[name]), (r, name)
            for name, got in zip(GRAD_KEYS, b):
                assert _bits_equal(got, cb[name].view(got.shape)), (r, name)
        else:
            assert all(t.numel() == 0 for t in f[:4]) and b[0].numel() == 0
            assert all(float(t.abs().sum()) == 0 for t in b[1:])
            for name in ("gw1", "gb1", "gw2", "gb2", "gw3", "gb3"):
                assert float(cb[name].abs().sum()) == 0
    # statistics, counts and running statistics: the same bits on every rank
    for f in fw[1:]:
        assert torch.equal(f[4], fw[0][4]) and torch.equal(f[5], fw[0][5])
    assert torch.equal(fw[0][5], torch.full((3,), float(maps * h * w), dtype=torch.float64, device=DEV))
    ref = _oracle(c, weights, params)
    moved = []
    for f in fw:
        block = copy.deepcopy(ref)
        norms_r = [block.layers.abn_down_project[0], block.layers.abn[0], block.layers.abn_up_project[0]]
        for i, (bn, (o, k)) in enumerate(zip(norms_r, bk._stats_slices(c // 2, c))):
            BN.update_running_stats(bn, f[4][o:o + k], f[4][o + k:o + 2 * k], f[5][i:i + 1])
        moved.append(list(block.buffers()))
    for bufs in moved[1:]:
        assert all(torch.equal(a, b) for a, b in zip(bufs, moved[0]))
    if maps * h * w < 900:
        # with few values per channel, one ReLU mask flipped by the kernels' TF32 operand rounding moves a norm's gradient sums by
        # O(1 / sqrt(n)), far past torch's fp32 error: such shapes are checked against the chain above only
        return
    # the whole batch against the fp64 oracle, within the Bottleneck tests' bar
    r64, m64 = _oracle_step(ref, x, g, torch.float64)
    r32, m32 = _oracle_step(ref, x, g, torch.float32)
    got = [torch.cat([f[0] for f in fw]), torch.cat([b[0] for b in bw])]
    got += [sum(b[k] for b in bw) for k in (1, 2, 3, 4, 5, 6, 7, 8, 9)]                # each rank's own gradients add up
    names = ["out", "x"] + [n for n, _ in m64.named_parameters()]
    order = [0, 1] + [2 + [n for n, _ in m64.named_parameters()].index(k) for k in (
        "layers.conv_down_project.weight", "layers.conv.weight", "layers.conv_up_project.weight", "layers.abn_down_project.0.weight",
        "layers.abn_down_project.0.bias", "layers.abn.0.weight", "layers.abn.0.bias", "layers.abn_up_project.0.weight",
        "layers.abn_up_project.0.bias")]
    for a, k in zip(got, order):
        e, e_ref = _rel(a, r64[k]), _rel(r32[k], r64[k])
        assert e <= max(3 * e_ref, 1e-3), (names[k], e, e_ref)
    for a, b64, b32 in zip(moved[0], m64.buffers(), m32.buffers()):
        if a.is_floating_point():
            assert _rel(a, b64) <= max(3 * _rel(b32, b64), 1e-3)
        else:
            assert int(a) == int(b64) == 1


def test_padding_is_the_normalized_maps_under_a_group():
    """bn1 and bn2 with weight 0 and bias 1 (tests/test_bottleneck_gpu.py's case) over two ranks: relu(bn(y)) is 1 on the maps and the
    3x3 padding and the 1x1 tiles' tails must stay 0, as the chain of the group entry points computes them"""
    x, weights, norms = operands(3, 35, 7, 12, seed=3)
    params = _affine(norms)
    for i in (0, 2):
        params[i] = torch.zeros_like(params[i])
        params[i + 1] = torch.ones_like(params[i + 1])
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(8)).to(DEV)
    shards, gouts = torch.split(x, [1, 2]), torch.split(g, [1, 2])
    fw, bw = _sync(shards, gouts, weights, params)
    chain_f = _lockstep([_chain_forward(xr, weights, params) for xr in shards])
    chain_b = _lockstep([_chain_backward(gr, xr, weights, params, f) for xr, gr, f in zip(shards, gouts, chain_f)])
    for f, b, cf, cb in zip(fw, bw, chain_f, chain_b):
        for name, got in (("y2", f[2]), ("y3", f[3]), ("out", f[0])):
            assert _bits_equal(got, cf[name]), name
        for name in ("gW_conv", "gW_up"):
            got = b[GRAD_KEYS.index(name)]
            assert _bits_equal(got, cb[name].view(got.shape)), name


def test_each_gradient_alone(monkeypatch):
    """each of the 10 gradients asked for alone, over three ranks (one empty), into NaN-filled memory between sentinels: the full
    run's bits, None for the others, the margins intact, and ``sync_stages`` gathers"""
    x, weights, norms = operands(4, 35, 7, 12, seed=5)
    params = _affine(norms)
    g = torch.randn(x.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    sizes = [1, 0, 3]
    shards, gouts = torch.split(x, sizes), torch.split(g, sizes)
    fw, full = _sync(shards, gouts, weights, params)
    bufs = []
    make = bk._grad_outputs

    def nan_outputs(*args):
        def fill(t):
            if t is None:
                return None
            view, buf = nan_filled(*t.shape)
            bufs.append(buf)
            return view
        gx, gwd, gwc, gwu, gn = make(*args)
        return fill(gx), fill(gwd), fill(gwc), fill(gwu), [fill(t) for t in gn]
    monkeypatch.setattr(bk, "_grad_outputs", nan_outputs)
    expected_gathers = (3, 3, 2, 1, 2, 2, 1, 1, 0, 0)
    for k in range(10):
        need = [j == k for j in range(10)]
        bufs.clear()
        calls = [[] for _ in shards]
        bw = _lockstep([_counting(bk.sync_backward_stages(gr, xr, *f[1:5], *weights, params, EPS, need), cl)
                        for xr, gr, f, cl in zip(shards, gouts, fw, calls)])
        assert all(len(cl) == expected_gathers[k] for cl in calls), (GRAD_KEYS[k], [len(cl) for cl in calls])
        for r, (b, fb) in enumerate(zip(bw, full)):
            assert all(gi is None for j, gi in enumerate(b) if j != k)
            assert _bits_equal(b[k], fb[k]), (r, GRAD_KEYS[k])
        assert bufs and all(margins_intact(buf) for buf in bufs)


# ------------------------------------------------------------------------------------------------------------------------------
# the module
# ------------------------------------------------------------------------------------------------------------------------------
def _blocks(c=64, seed=0):
    """(a TensorCoreBottleneck over BatchNorm2d norms, the same over FusedSyncBatchNorm norms), equal parameters and buffers"""
    from tests.test_bottleneck_gpu import _block
    plain = bk.TensorCoreBottleneck.from_module(_block(c, seed)).to(DEV)
    synced = nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    for abn in (synced.layers.abn_down_project, synced.layers.abn, synced.layers.abn_up_project):
        abn[0] = BN.FusedSyncBatchNorm(abn[0])
    return plain, synced


def _module_step(module, x, g, amp=False):
    for p in module.parameters():
        p.grad = None
    xi = x.detach().clone().requires_grad_(True)
    with torch.autocast("cuda", enabled=amp):
        out = module(xi)
    out.float().backward(g)
    return [out, xi.grad] + [p.grad for p in module.parameters()] + list(module.buffers())


@pytest.mark.parametrize("case", ["eval", "train-world-1", "train-amp-group-of-one"])
def test_module_matches_the_unsynced_operator_bit_for_bit(case, monkeypatch):
    """eval and a world of one run the unsynced operator; a group of one (SyncBottleneck with a one-rank gather) computes the same
    bits, under autocast too"""
    plain, synced = _blocks()
    x = torch.randn(3, 64, 20, 24, device=DEV)
    g = torch.randn(3, 64, 20, 24, device=DEV)
    amp = "amp" in case
    if amp:
        x = x.half()
        calls = []
        monkeypatch.setattr(bk, "sync_group", lambda norm: "group")
        monkeypatch.setattr(bk, "gather", lambda t, group: calls.append(group) or t[None])
    if case == "eval":
        plain.eval()
        synced.eval()
    ref, got = _module_step(plain, x, g, amp), _module_step(synced, x, g, amp)
    assert got[0].dtype == torch.float32 and got[1].dtype == x.dtype
    for i, (a, b) in enumerate(zip(got, ref)):
        assert a.dtype == b.dtype and torch.equal(a, b), i
    if amp:
        assert calls == ["group"] * 6


# ------------------------------------------------------------------------------------------------------------------------------
# two processes on one GPU over gloo
# ------------------------------------------------------------------------------------------------------------------------------
C, X, Y, T_FUT, LATENT = 16, 12, 16, 3, 8
BATCH = (2, 1)                                               # per-rank batch: uneven


def _inputs():
    g = torch.Generator().manual_seed(11)
    zs = [torch.randn(bb, T_FUT, LATENT, X, Y, generator=g) for bb in BATCH]
    hs = [torch.randn(bb, C, X, Y, generator=g) for bb in BATCH]
    return zs, hs


def _model():
    torch.manual_seed(0)
    return FuturePrediction(C, LATENT, n_gru_blocks=3, n_res_layers=3)


def _loss(out):
    return (out * out.detach().cos()).sum()


def _worker(rank, world, port, backend, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        from fiery_b200 import install
        dev = torch.device("cuda", rank % torch.cuda.device_count())
        torch.cuda.set_device(dev)
        ref = nn.SyncBatchNorm.convert_sync_batchnorm(_model()).to(dev).train()
        holder = nn.Module()
        holder.future_prediction = copy.deepcopy(ref)
        install.use_fused_sync_batch_norm(holder)
        install.use_tensor_core_future_prediction(holder)
        install.use_tensor_core_sync_bottlenecks(holder)
        mine = holder.future_prediction
        plain = sum(type(m) is nn.SyncBatchNorm for m in mine.modules())
        blocks = sum(isinstance(m, bk.TensorCoreBottleneck) for m in mine.modules())
        zs, hs = _inputs()
        z, h0 = zs[rank].to(dev), hs[rank].to(dev)

        def run(m):
            zi, hi = z.clone().requires_grad_(True), h0.clone().requires_grad_(True)
            out = m(zi, hi)
            _loss(out).backward()
            grads = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
            for v in grads.values():
                dist.all_reduce(v)
                v /= world
            return [out.detach(), zi.grad, hi.grad], grads, {n: bf.clone() for n, bf in m.named_buffers()}
        o_ref, g_ref, s_ref = run(ref)
        real = {name: getattr(dist, name) for name in ("all_gather", "all_gather_into_tensor")}
        calls = [0]

        def counted(fn):
            def call(*a, **k):
                calls[0] += 1
                return fn(*a, **k)
            return call
        for name, fn in real.items():                   # gloo gathers with all_gather, NCCL with all_gather_into_tensor
            setattr(dist, name, counted(fn))
        try:
            o, gr, st = run(mine)
        finally:
            for name, fn in real.items():
                setattr(dist, name, fn)
        expected = 2 * 3 * blocks + 2 * 3 * T_FUT       # 3 per Bottleneck each way, 1 per GRU step each way
        host = lambda ts: [t.cpu().numpy() for t in ts]                                     # noqa: E731
        hostd = lambda d: {k: v.cpu().numpy() for k, v in d.items()}                        # noqa: E731
        q.put((rank, host(o), host(o_ref), hostd(gr), hostd(g_ref), hostd(st), hostd(s_ref), calls[0], expected, plain, blocks))
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
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    dev = lambda x: [torch.from_numpy(a) for a in x] if isinstance(x, list) else {k: torch.from_numpy(a) for k, a in x.items()}  # noqa
    return [(r[0], *[dev(x) for x in r[1:7]], *r[7:]) for r in res]


def _whole_batch_fp64(tf32_operands=False):
    """the group's computation in one process: the model with plain BatchNorms, fp64, on the ranks' shards concatenated (with
    ``tf32_operands`` every convolution, the GRUs' and the Bottlenecks', takes TF32-rounded operands, as the kernels do): each rank's
    slice of the output and input gradients, the parameter gradients over the ranks' mean loss, and the running statistics"""
    from tests.test_spatial_gru_gpu import _tf32_operands
    m = _model().cuda().double().train()
    if tf32_operands:
        _tf32_operands(m)
    zs, hs = _inputs()
    z, h0 = (torch.cat(t).cuda().double().requires_grad_(True) for t in (zs, hs))
    out = m(z, h0)
    _loss(out).backward()
    grads = {n: p.grad.cpu() / len(BATCH) for n, p in m.named_parameters()}
    cuts = [0] + list(torch.tensor(BATCH).cumsum(0))
    per_rank = [[t.detach().cpu()[cuts[r]:cuts[r + 1]] for t in (out, z.grad, h0.grad)] for r in range(len(BATCH))]
    return per_rank, grads, {n: bf.cpu() for n, bf in m.named_buffers()}


def _check(res):
    from tests.test_sync_batch_norm_gpu import _within
    o64s, g64, s64 = _whole_batch_fp64()
    ot64s, gt64, st64 = _whole_batch_fp64(tf32_operands=True)
    for rank, o, o_ref, gr, g_ref, st, s_ref, n_gather, expected, plain, blocks in res:
        assert plain == 0 and blocks == 9
        assert n_gather == expected, (rank, n_gather, expected)
        for i in range(3):
            assert _within(o[i], o_ref[i], o64s[rank][i], ot64s[rank][i]), (rank, i)
        assert set(gr) == set(g_ref)
        for k in g_ref:
            assert _within(gr[k], g_ref[k], g64[k], gt64[k]), (rank, k, _rel(gr[k], g64[k]), _rel(g_ref[k], g64[k]))
        for k in s_ref:
            if s_ref[k].is_floating_point():
                assert _within(st[k], s_ref[k], s64[k], st64[k]), k
            else:
                assert torch.equal(st[k], s_ref[k]), k
    for k in res[0][5]:                                # the running statistics: bit for bit the same on both ranks
        assert torch.equal(res[0][5][k], res[1][5][k]), k


def test_two_processes_over_gloo():
    _check(_spawn("gloo"))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL needs one GPU per rank")
def test_two_processes_over_nccl():
    _check(_spawn("nccl"))
