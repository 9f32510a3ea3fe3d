"""GPU: the temporal block's tail across the range its C ABI and ``aggregation_reason`` accept -- ``temporal_aggregation`` (the entry's
kernels in swapped roles, csrc/temporal_entry.cu) and the spatial sums (csrc/spatial_sums.cu) -- with the cases and rules of
tests/_temporal_cases.py.

A  every AGG_CASES case (temporal_aggregation_kernel<1> and <2>, the no-bias kernel for R = 0, grad_paths'
   temporal_entry_fwd_kernel<1..4>, the weight gradient's nc 1 and 2 at 128 .. 512 threads, every ring depth; maps of a partial
   tile, one tile, one over, one under and 40000 pixels) through the C ABI into guarded buffers from NaN-poisoned inputs, bit-exact on
   small integers against fp64;
B  the forward of one batch element does not depend on its neighbours;
C  operand rounding: the packed path columns to nearest, the paths as the tensor core reads them, the pooled bias unrounded, and the
   backward's pooled terms against fp64 within their fp32 rounding bound;
D  the spatial sums bit for bit against tests/_temporal_cases.spatial_sums_model: the loop edges, aligned and misaligned planes, NaN
   gap planes, the copy route;
E  one shape whose offsets pass 2^31 elements;
F  the host routes: an X*Y the kernel does not take, a sliced path, gradients for some paths only, an expanded output gradient, fp16
   under autocast;
G  whole TemporalModels wider than the shipped one (EXTRA_IN_CHANNELS > 0, START_OUT_CHANNELS = 128) against the fp64 oracle."""
import contextlib
import copy
import warnings

import pytest
import torch

from fiery_b200 import _lib, install, ops, temporal  # noqa: F401  (registers the operators)
from fiery_b200.temporal import TensorCorePyramidPooling, TensorCoreTemporalBlock, _ptrs, aggregation_backward, \
    aggregation_forward, pack_aggregation, spatial_sums
from oracle import temporal_oracle as TO
from tests import _temporal_cases as TC
from tests.test_temporal_envelope_gpu import _device_ints, _Entry, _ints, _need_memory, _stream, _which
from tests.test_temporal_tail_cpu import _holder
from tests.test_temporal_tail_gpu import SUM_GRIDS, _agg_reference, _model, _nerr, _no_tf32, _Recorder, _step, \
    _sums_guarded  # noqa: F401  (_no_tf32: the module's fixture)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
_ids = lambda v: str(v).replace(" ", "")
U = 2.0 ** -24                                     # fp32 unit roundoff


@contextlib.contextmanager
def _deterministic():
    """uninitialised outputs are NaN-filled, so an element the kernels never write shows up"""
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)


def _op(paths, weight, pooled):
    return torch.ops.fiery_b200.temporal_aggregation(paths, weight, pooled)


# ------------------------------------------------------------------------------------------------------------------------------
# A: every case through the C ABI, guarded
# ------------------------------------------------------------------------------------------------------------------------------
def _swapped_entry(grad, weight, paths):
    """The entry in swapped roles on guarded buffers: x = the aggregation's output gradient (b, N, s, X, Y), the convolutions the
    path columns A_q transposed; its pack is the aggregation's."""
    n, c = int(weight.shape[0]), sum(paths)
    a_t = weight.reshape(n, -1)[:, :c].t()
    return _Entry(grad, [t[..., None, None, None] for t in a_t.split(list(paths))], None, "channel_major")


def _forward_guarded(e, paths, bias):
    """fiery_temporal_aggregation_forward of poisoned paths and bias (b, s, N) (None: NULL) into an output between sentinel margins
    of 64 pixels per channel"""
    b, n, s, h, w = e.x.shape
    buf, out = TC.guarded(b * n * s * h * w, 64 * n, 64 * n, DEV)
    ps = [TC.poisoned(p, DEV) for p in paths]
    bp = TC.poisoned(bias, DEV).data_ptr() if bias is not None else 0
    _lib.check(e.lib.fiery_temporal_aggregation_forward(e.d, _ptrs(ps), e.pack.data_ptr(), bp, out.data_ptr(), _stream()),
               "aggregation forward")
    TC.assert_written_and_contained(buf, out, "output")
    return out.view(b, n, s, h, w)


@pytest.mark.parametrize("n,paths,r,grid,b,s", TC.AGG_CASES, ids=_ids)
def test_every_aggregation_case_guarded_and_bit_exact(n, paths, r, grid, b, s):
    """Forward through fiery_temporal_aggregation_forward (the pack in a buffer of exactly its size, equal to pack_aggregation's),
    grad_paths and the path columns of the weight gradient through the entry's C ABI in swapped roles, all guarded; the host's
    forward and backward the same bits; the weight gradient's bits whatever its workspace held."""
    gen = torch.Generator().manual_seed(TC.AGG_CASES.index((n, paths, r, grid, b, s)))
    ps = [_ints(gen, b, c, s, *grid).to(DEV) for c in paths]
    weight, pooled = _ints(gen, n, sum(paths) + r, 1, 1, 1).to(DEV), _ints(gen, b, r, s).to(DEV)
    grad = _ints(gen, b, n, s, *grid).to(DEV)
    z_ref, gp_ref, gw_ref, gv_ref = _agg_reference(ps, weight, pooled, grad)
    c = sum(paths)

    e = _swapped_entry(grad, weight, paths)
    assert torch.equal(e.pack.view(torch.int32), pack_aggregation(weight, tuple(paths)).view(torch.int32)), "pack"
    bias = torch.einsum("nr,brt->btn", weight.reshape(n, -1)[:, c:].double(), pooled.double()).float() if r else None
    z = _forward_guarded(e, ps, bias)
    assert torch.equal(z.double(), z_ref), "forward"
    assert torch.equal(aggregation_forward(ps, weight, pooled), z), "forward through the host"

    with _deterministic():
        gp, gw, gv = aggregation_backward(grad, ps, weight, pooled, True, True, True)
    for q, (a, ref) in enumerate(zip(gp, gp_ref)):
        assert torch.equal(a.double(), ref), f"grad_paths[{q}]"
    assert torch.equal(gw.double(), gw_ref), "grad_weight"
    assert torch.equal(gv.double(), gv_ref), "grad_pooled"

    for q, (a, ref) in enumerate(zip(e.forward(), gp_ref)):                 # grad_paths, guarded
        assert torch.equal(a.double(), ref), f"grad_paths[{q}] through the C ABI"
    first = e.backward_weight(ps)                                           # (sum C_q, N): the path columns, transposed
    assert torch.equal(first.double(), gw_ref.reshape(n, -1)[:, :c].t()), "weight gradient through the C ABI"
    for fill in (0.0, 1e30):                                                # the same bits whatever the workspace held
        assert torch.equal(e.backward_weight(ps, fill), first), fill


# ------------------------------------------------------------------------------------------------------------------------------
# B: batch and neighbour invariance
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,paths,r", [(64, (35, 35, 35), 23), (128, (48, 48, 48), 42)], ids=_ids)
def test_forward_of_a_batch_element_is_its_own(n, paths, r):
    gen = torch.Generator().manual_seed(n)
    ps = [torch.randn((3, c, 2, 12, 11), generator=gen).to(DEV) for c in paths]
    weight = (torch.randn((n, sum(paths) + r, 1, 1, 1), generator=gen) / 16).to(DEV)
    pooled = torch.randn((3, r, 2), generator=gen).to(DEV)
    z = aggregation_forward(ps, weight, pooled)
    for i in range(3):
        assert torch.equal(aggregation_forward([p[i:i + 1] for p in ps], weight, pooled[i:i + 1]), z[i:i + 1]), i


# ------------------------------------------------------------------------------------------------------------------------------
# C: operand rounding
# ------------------------------------------------------------------------------------------------------------------------------
ROUNDING = [(64, (35, 35, 35)), (128, (57, 64, 3, 100)), (33, (65, 63)), (96, (1, 8, 8))]


@pytest.mark.parametrize("n,paths", ROUNDING, ids=_ids)
def test_path_columns_are_packed_rounded_to_nearest(n, paths):
    """Path channel c holds a single 1.0, at pixel c: out[o, pixel c] = A[o, c] as packed.  An output gradient with a single 1.0 per
    channel, channel o at pixel o: grad_paths[c, pixel o] = A[o, c] from the same pack."""
    c, r = sum(paths), 3
    w = TC.full_mantissa((n, c + r), seed=n + c)
    want = TC.tf32_rna(w[:, :c])
    x = torch.zeros(1, c, 1, 256)
    x[0, torch.arange(c), 0, torch.arange(c)] = 1.0
    ps = [t.reshape(1, -1, 1, 16, 16).to(DEV) for t in x.split(list(paths), 1)]
    weight, pooled = w.reshape(n, c + r, 1, 1, 1).to(DEV), torch.zeros(1, r, 1, device=DEV)
    z = aggregation_forward(ps, weight, pooled).flatten(3).cpu()
    assert torch.equal(z[0, :, 0, :c], want) and int(torch.count_nonzero(z[0, :, 0, c:])) == 0
    g = torch.zeros(1, n, 1, 256)
    g[0, torch.arange(n), 0, torch.arange(n)] = 1.0
    gp, _, _ = aggregation_backward(g.reshape(1, n, 1, 16, 16).to(DEV), ps, weight, pooled, True, False, False)
    gp = torch.cat(gp, 1).flatten(3).cpu()
    assert torch.equal(gp[0, :, 0, :n], want.t()) and int(torch.count_nonzero(gp[0, :, 0, n:])) == 0


@pytest.mark.parametrize("n,paths", [(64, (35, 35, 35)), (128, (64, 64, 64, 64)), (96, (65, 63))], ids=_ids)
def test_paths_and_output_gradient_as_the_tensor_core_reads_them(n, paths):
    """A weight with a single 1.0 per output row, at a different path channel each: the output is those path channels as the tensor
    core reads fp32 from shared memory, and grad_paths the output gradient as the forward kernel reads it -- each uniformly rounded to
    nearest or uniformly truncated (NCHK 1 and 2 for the aggregation)."""
    c = sum(paths)
    m, b, s, grid = min(n, c), 2, 2, (8, 12)
    perm = torch.randperm(c, generator=torch.Generator().manual_seed(c))[:m]
    w = torch.zeros(n, c + 1)
    w[torch.arange(m), perm] = 1.0
    x = TC.full_mantissa((b, c, s, *grid), seed=n + c)
    ps = [t.contiguous().to(DEV) for t in x.split(list(paths), 1)]
    weight, pooled = w.reshape(n, c + 1, 1, 1, 1).to(DEV), torch.zeros(b, 1, s, device=DEV)

    def fwd(rnd):
        y = torch.zeros(b, n, s, *grid)
        y[:, :m] = rnd(x)[:, perm]
        return y
    _which(aggregation_forward(ps, weight, pooled), fwd, f"temporal aggregation (N = {n}), paths")
    g = TC.full_mantissa((b, n, s, *grid), seed=n + c + 1)
    gp, _, _ = aggregation_backward(g.to(DEV), ps, weight, pooled, True, False, False)

    def bwd(rnd):
        gx = torch.zeros(b, c, s, *grid)
        gx[:, perm] = rnd(g)[:, :m]
        return gx
    _which(torch.cat(gp, 1), bwd, f"temporal aggregation grad_paths (N = {n}), grad")


@pytest.mark.parametrize("n,paths,r", [(64, (35, 35, 35), 23), (128, (48, 48, 48), 42), (7, (8,), 1)], ids=_ids)
def test_pooled_bias_is_added_unrounded(n, paths, r):
    """Zero path columns and a single 1.0 per output row in the pooled columns: every output pixel is its pooled value, which the
    bias carries in fp32 -- not rounded to TF32 on the way."""
    c, b, s, grid = sum(paths), 2, 3, (4, 17)
    w = torch.zeros(n, c + r)
    w[torch.arange(n), c + torch.arange(n) % r] = 1.0
    ps = [TC.full_mantissa((b, q, s, *grid), seed=q).to(DEV) for q in paths]
    pooled = TC.full_mantissa((b, r, s), seed=n + r)
    assert not torch.equal(TC.tf32_rna(pooled), pooled)
    z = aggregation_forward(ps, w.reshape(n, c + r, 1, 1, 1).to(DEV), pooled.to(DEV))
    want = pooled[:, torch.arange(n) % r][..., None, None].expand(b, n, s, *grid)
    assert torch.equal(z.cpu(), want)


def _gamma(k):
    return k * U / (1 - k * U)


@pytest.mark.parametrize("n,paths,r,grid", [(64, (35, 35, 35), 23, (52, 48)), (128, (48, 48, 48), 42, (20, 51))], ids=_ids)
def test_pooled_gradients_are_fp32_sums_of_the_spatial_sums(n, paths, r, grid):
    """grad_pooled = W_P^T G and the pooled columns of grad_weight = sum over frames of G pooled^T, with G the output gradient's
    spatial sums: G is the kernel's (bit for bit the order model), the rest fp32 products summed, so each element is within
    gamma_{k+1} * sum |products| of fp64 on the same G (k summands)."""
    c, b, s = sum(paths), 2, 3
    g = TC.full_mantissa((b, n, s, *grid), seed=n)
    w = TC.full_mantissa((n, c + r), seed=n + 1) / 64
    pooled = TC.full_mantissa((b, r, s), seed=n + 2)
    ps = [TC.full_mantissa((b, q, s, *grid), seed=q).to(DEV) for q in paths]
    _, gw, gv = aggregation_backward(g.to(DEV), ps, w.reshape(n, c + r, 1, 1, 1).to(DEV), pooled.to(DEV), False, True, True)
    sums = torch.from_numpy(TC.spatial_sums_model(g.flatten(3).numpy(), grid[0] * grid[1]))
    assert torch.equal(spatial_sums(g.to(DEV)).cpu(), sums)
    G, WP, V = sums.double(), w[:, c:].double(), pooled.double()
    checks = [("grad_pooled", gv, torch.einsum("nr,bnt->brt", WP, G), torch.einsum("nr,bnt->brt", WP.abs(), G.abs()), n),
              ("grad_weight pooled columns", gw.reshape(n, -1)[:, c:], torch.einsum("bnt,brt->nr", G, V),
               torch.einsum("bnt,brt->nr", G.abs(), V.abs()), b * s)]
    for what, got, ref, mag, k in checks:
        err = (got.cpu().double() - ref).abs()
        bound = _gamma(k + 1) * mag
        assert bool((err <= bound).all()), f"{what}: {float((err / bound).max()):.2f} x the bound"


# ------------------------------------------------------------------------------------------------------------------------------
# D: spatial sums against the order model
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", [0, 1, 2], ids=["aligned", "offset1", "offset2"])
@pytest.mark.parametrize("grid", SUM_GRIDS, ids=str)
def test_sums_equal_the_order_model_bitwise(grid, offset):
    """Planes at a 16-byte-aligned pitch with NaN between them, every base aligned (float4 loads) or none (scalar loads)"""
    b, c, s, p = 2, 5, 3, grid[0] * grid[1]
    gen = torch.Generator().manual_seed(p + offset)
    x = torch.randn((b, c, s, p), generator=gen) * torch.exp2(torch.randint(-8, 9, (b, c, s, p), generator=gen).float())
    pitch = (p + 3) // 4 * 4 + 4
    buf = torch.full((b * c * s * pitch + 8,), float("nan"), device=DEV)
    view = buf[offset:offset + b * c * s * pitch].view(b, c, s, pitch)[..., :p].view(b, c, s, *grid)
    view.copy_(x.view(b, c, s, *grid))
    got, guards = _sums_guarded(view)
    assert guards
    assert torch.equal(got.cpu(), torch.from_numpy(TC.spatial_sums_model(x.numpy(), p)))


@pytest.mark.parametrize("grid", [(3, 341), (17, 241), (52, 49), (1, 3)], ids=str)
def test_sums_of_frame_major_planes_with_nan_gaps(grid):
    gen = torch.Generator().manual_seed(grid[1])
    x = torch.randn((2, 9, 3, *grid), generator=gen)
    got = spatial_sums(TC.poisoned_frame_major(x, DEV)).cpu()
    assert bool(torch.isfinite(got).all())
    assert torch.equal(got, torch.from_numpy(TC.spatial_sums_model(x.flatten(3).numpy(), grid[0] * grid[1])))


@pytest.mark.parametrize("kind", ["fp16", "bf16", "channels_last_3d"])
def test_sums_copy_route(kind):
    x = torch.randn((2, 6, 3, 17, 241), generator=torch.Generator().manual_seed(5)).to(DEV)
    xin = {"fp16": x.half(), "bf16": x.bfloat16(), "channels_last_3d": x.contiguous(memory_format=torch.channels_last_3d)}[kind]
    up = xin.float().contiguous()
    want = torch.from_numpy(TC.spatial_sums_model(up.flatten(3).cpu().numpy(), 17 * 241))
    for got in (spatial_sums(xin), torch.ops.fiery_b200.spatial_sums(xin)):
        assert got.dtype == torch.float32 and torch.equal(got.cpu(), want)


# ------------------------------------------------------------------------------------------------------------------------------
# E: offsets past 2^31 elements
# ------------------------------------------------------------------------------------------------------------------------------
def test_aggregation_offsets_past_2_31_elements():
    """N = 64 from one 8-channel path and R = 4 pooled channels over 3 x 3 frames of 2048 x 2048: the output has 2.4 G elements, so
    b * sb + k * sc passes 2^31.  References per (batch, frame) slice, fp32 matrix products, exact on small integers."""
    _need_memory(16)
    n, c, r, b, s, X, Y = 64, 8, 4, 3, 3, 2048, 2048
    gen = torch.Generator(device=DEV).manual_seed(2)
    p, weight, pooled = _device_ints(gen, b, c, s, X, Y), _device_ints(gen, n, c + r, 1, 1, 1), _device_ints(gen, b, r, s)
    a, wp = weight.view(n, c + r)[:, :c], weight.view(n, c + r)[:, c:]
    y = aggregation_forward([p], weight, pooled)
    assert y.numel() > 2 ** 31
    for bb in range(b):
        for t in range(s):
            want = a @ p[bb, :, t].reshape(c, -1) + (wp @ pooled[bb, :, t])[:, None]
            assert torch.equal(y[bb, :, t].reshape(n, -1), want), (bb, t)
            del want
    for bb in range(b):                                        # the output-sized tensor becomes the output gradient
        y[bb].random_(-2, 3, generator=gen)
    (gp,), gw, gv = aggregation_backward(y, [p], weight, pooled, True, True, True)
    sums = spatial_sums(y)
    gw_ref = torch.zeros((n, c), dtype=torch.float64, device=DEV)
    for bb in range(b):
        for t in range(s):
            g = y[bb, :, t].reshape(n, -1)
            assert torch.equal(gp[bb, :, t].reshape(c, -1), a.t() @ g), (bb, t)
            assert torch.equal(sums[bb, :, t].double(), g.sum(1, dtype=torch.float64)), (bb, t)
            gw_ref += (g @ p[bb, :, t].reshape(c, -1).t()).double()
            del g
    G = sums.double()
    assert torch.equal(gw.view(n, c + r)[:, :c].double(), gw_ref), "weight gradient, path columns"
    assert torch.equal(gw.view(n, c + r)[:, c:].double(), torch.einsum("bnt,brt->nr", G, pooled.double())), "pooled columns"
    assert torch.equal(gv.double(), torch.einsum("nr,bnt->brt", wp.double(), G)), "grad_pooled"
    del p, y, gp
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------------
# F: host routes
# ------------------------------------------------------------------------------------------------------------------------------
def test_uncovered_pixel_count_runs_the_concat_aggregation_with_one_warning(monkeypatch):
    """A model built for a 51 x 49 map: the pooling covers the map, but X*Y = 2499 is not a multiple of 4.  install leaves the blocks
    to the reference (the entry needs the same multiple), so a block adopted by the bare constructor is what reaches the
    aggregation's own check: it warns once and runs the concat and Conv3d, and the step still matches fp64."""
    monkeypatch.setattr(_lib, "_warned", set())
    grid = (51, 49)
    ref = _model(3, 0, seed=5, grid=grid)
    sw = copy.deepcopy(ref)
    with pytest.warns(RuntimeWarning, match="X\\*Y = 2499"):
        install.use_tensor_core_temporal_model(_holder(sw))
    assert not any(isinstance(b, TensorCoreTemporalBlock) for b in sw.model)
    for i, blk in enumerate(sw.model):
        sw.model[i] = TensorCoreTemporalBlock(blk)
    install.use_tensor_core_pyramid_pooling(_holder(sw))
    assert all(isinstance(b.pyramid_pooling, TensorCorePyramidPooling) for b in sw.model)
    for m in (ref, sw):
        m.train(True)
    ref64 = copy.deepcopy(ref).double()
    gen = torch.Generator().manual_seed(6)
    bev, ego = torch.randn((2, 3, 64, *grid), generator=gen).to(DEV), torch.randn((2, 3, 6), generator=gen).to(DEV)
    gout = torch.randn((2, 1, 64, *grid), generator=gen).to(DEV)
    y64, gx64, gp64 = _step(ref64, bev.double(), ego.double(), gout.double(), "concat")
    y0, gx0, gp0 = _step(ref, bev, ego, gout, "concat", tf32=True)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        y1, gx1, gp1 = _step(sw, bev, ego, gout, "concat")
        with _Recorder() as disp:
            _step(sw, bev, ego, gout, "concat")
    msgs = [str(w.message) for w in rec]
    assert sum("aggregation on X*Y = 2499" in m for m in msgs) == 1, msgs
    assert sum("input of X*Y = 2499" in m for m in msgs) == 1, msgs
    names = [name for name, _, _ in disp.ops]
    assert "temporal_aggregation" not in names and "spatial_sums" in names
    for what, a, r, o in [("out", y1, y64, y0), ("grad_bev", gx1, gx64, gx0)] + [(k, gp1[k], gp64[k], gp0[k]) for k in gp64]:
        assert _nerr(a, r) <= max(3 * _nerr(o, r), 1e-5), f"{what}: {_nerr(a, r):.3e} vs oracle {_nerr(o, r):.3e}"


def _op_case(seed, b=2, s=3, grid=(8, 12), paths=(35, 35, 35), n=64, r=23):
    gen = torch.Generator().manual_seed(seed)
    ps = [torch.randn((b, c, s, *grid), generator=gen).to(DEV) for c in paths]
    weight = (torch.randn((n, sum(paths) + r, 1, 1, 1), generator=gen) / 11).to(DEV)
    return ps, weight, torch.randn((b, r, s), generator=gen).to(DEV), torch.randn((b, n, s, *grid), generator=gen).to(DEV)


def _op_step(paths, weight, pooled, grad, need=None):
    """forward and backward of the operator; need[q]: path q requires grad (all by default).  Returns (z, [grad_paths], grad_weight,
    grad_pooled)."""
    need = need or [True] * len(paths)
    pi = [p.detach().requires_grad_(k) for p, k in zip(paths, need)]
    wi, vi = weight.detach().requires_grad_(True), pooled.detach().requires_grad_(True)
    z = _op(pi, wi, vi)
    z.backward(grad)
    return z.detach(), [p.grad for p in pi], wi.grad, vi.grad


def _assert_same_bits(got, want):
    z, gp, gw, gv = got
    z0, gp0, gw0, gv0 = want
    assert torch.equal(z, z0) and torch.equal(gw, gw0) and torch.equal(gv, gv0)
    for a, b in zip(gp, gp0):
        assert (a is None) == (b is None) and (a is None or torch.equal(a, b))


def test_sliced_path_gives_the_bits_of_its_contiguous_copy():
    ps, weight, pooled, grad = _op_case(seed=1)
    wide = torch.randn((2, 40, 3, 8, 12), generator=torch.Generator().manual_seed(2)).to(DEV)
    sliced = wide[:, 3:38]
    assert not sliced.is_contiguous()
    _assert_same_bits(_op_step([ps[0], sliced, ps[2]], weight, pooled, grad),
                      _op_step([ps[0], sliced.contiguous(), ps[2]], weight, pooled, grad))


def test_gradients_for_some_paths_only():
    ps, weight, pooled, grad = _op_case(seed=3)
    z, gp, gw, gv = _op_step(ps, weight, pooled, grad)
    for need in ([True, False, True], [False, True, False], [False, False, True]):
        got = _op_step(ps, weight, pooled, grad, need)
        _assert_same_bits(got, (z, [g if k else None for g, k in zip(gp, need)], gw, gv))


def test_expanded_output_gradient_gives_the_bits_of_its_contiguous_copy():
    ps, weight, pooled, _ = _op_case(seed=4)
    g = torch.randn((1, 64, 1, 1, 12), generator=torch.Generator().manual_seed(5)).to(DEV).expand(2, 64, 3, 8, 12)
    assert g.stride()[0] == 0
    _assert_same_bits(_op_step(ps, weight, pooled, g), _op_step(ps, weight, pooled, g.contiguous()))


def test_fp16_paths_under_autocast():
    ps, weight, pooled, grad = _op_case(seed=6)
    ps16 = [p.half() for p in ps]
    z0, gp0, gw0, gv0 = _op_step([p.float() for p in ps16], weight, pooled, grad)
    pi = [p.detach().requires_grad_(True) for p in ps16]
    wi, vi = weight.detach().requires_grad_(True), pooled.detach().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16):
        z = _op(pi, wi, vi)
    assert z.dtype == torch.float32 and torch.equal(z, z0)
    z.backward(grad)
    for p, g0 in zip(pi, gp0):
        assert p.grad.dtype == torch.float16 and torch.equal(p.grad, g0.half())
    assert torch.equal(wi.grad, gw0) and torch.equal(vi.grad, gv0)


# ------------------------------------------------------------------------------------------------------------------------------
# G: whole models beyond the shipped width
# ------------------------------------------------------------------------------------------------------------------------------
# (receptive field, start_out_channels, extra_in_channels, which blocks the entry covers).  Block i takes 64 + (i - 1) * extra channels
# and gives 64 + i * extra, so its aggregation has N = 80, 96, 112: NCHK = 2 in real blocks.  With 128 start channels block 1 is
# 128 -> 144, whose entry would stack 3 x 64 + 144 = 336 > 256 output channels: it stays the reference's block, with one warning.
WIDE = [(3, 64, 16, (True, True)), (5, 64, 16, (True, True, True, True)), (3, 128, 16, (True, False))]
WIDE_GRID = (50, 52)          # 2600 pixels: a partial last tile of 64 and of 128 pixels; Y % 4 == 0, so the causal convs run too


@pytest.mark.parametrize("route", ["concat", "folded"])
@pytest.mark.parametrize("rf,start,extra,covered", WIDE, ids=_ids)
def test_wide_models_match_oracle(rf, start, extra, covered, route, monkeypatch):
    monkeypatch.setattr(_lib, "_warned", set())
    ref = _model(rf, 0, seed=rf + start, grid=WIDE_GRID, start_out_channels=start, extra_in_channels=extra)
    sw = copy.deepcopy(ref)
    h = _holder(sw)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        install.use_tensor_core_temporal_model(h)
        install.use_tensor_core_causal_convs(h)
        install.use_tensor_core_pyramid_pooling(h)
    msgs = [str(w.message) for w in rec]
    assert tuple(isinstance(b, TensorCoreTemporalBlock) for b in sw.model) == covered
    assert all(isinstance(b.pyramid_pooling, TensorCorePyramidPooling) for b in sw.model)
    if all(covered):
        assert msgs == []
    else:
        assert len(msgs) == 1 and "TemporalBlock(s) not covered" in msgs[0] and "N_out" in msgs[0], msgs
        assert all(f"block {i}:" in msgs[0] for i, cov in enumerate(covered) if not cov)
    for m in (ref, sw):
        m.train(True)
    ref64 = copy.deepcopy(ref).double()
    gen = torch.Generator().manual_seed(rf + start)
    bev, ego = torch.randn((2, rf, 64, *WIDE_GRID), generator=gen).to(DEV), torch.randn((2, rf, 6), generator=gen).to(DEV)
    gout = torch.randn((2, 1, ref.out_channels, *WIDE_GRID), generator=gen).to(DEV)
    y64, gx64, gp64 = _step(ref64, bev.double(), ego.double(), gout.double(), "concat")
    y0, gx0, gp0 = _step(ref, bev, ego, gout, "concat", tf32=True)
    with warnings.catch_warnings(record=True) as rec, _Recorder() as disp:
        warnings.simplefilter("always")
        y1, gx1, gp1 = _step(sw, bev, ego, gout, route)
    assert not [str(w.message) for w in rec if "fiery_b200" in str(w.message)]          # no swapped module falls back
    assert [name for name, _, _ in disp.ops].count("temporal_aggregation") == sum(covered)
    assert [name for name, _, _ in disp.ops].count("causal_conv3d") == 2 * len(covered)
    assert set(gp1) == set(gp0) == set(gp64)
    for what, a, r, o in [("out", y1, y64, y0), ("grad_bev", gx1, gx64, gx0)] + [(k, gp1[k], gp64[k], gp0[k]) for k in gp64]:
        assert _nerr(a, r) <= max(3 * _nerr(o, r), 1e-5), f"{what}: {_nerr(a, r):.3e} vs oracle {_nerr(o, r):.3e}"
