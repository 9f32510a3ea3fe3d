"""CPU: the case lists and references of tests/_temporal_cases.py, rehearsed before tests/test_temporal_envelope_gpu.py and
tests/test_temporal_tail_envelope_gpu.py spend GPU time on them -- which causal-convolution and aggregation kernels, instantiations
and ring depths the lists reach (and which the older lists do not), the grid classes and tile counts they were chosen for against the
C ABI's workspace sizes, the spatial sums' order model against fp64 and on values whose sum shows the order, TF32 rounding on
hand-picked bit patterns, and the by-indexing expectations against fp64 F.conv3d and its gradients."""
import math
import struct

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fiery_b200 import _lib
from tests import _temporal_cases as TC
from tests.test_temporal_entry_gpu import BLOCKS


def test_new_cases_reach_every_causal_conv_kernel_and_the_old_list_does_not():
    from tests.test_causal_conv_gpu import CASES as OLD
    new = TC.instantiations(TC.A_CASES)
    assert {(k, n) for k, n, _ in new} == TC.ALL_KERNELS and len(TC.ALL_KERNELS) == 24
    for kernel in ("forward", "dgrad"):
        assert {nks for k, _, nks in new if k == kernel} == set(range(1, 9)), kernel
    assert any(cin > cout for _, (cin, cout), *_ in TC.A_CASES) and any(cin < cout for _, (cin, cout), *_ in TC.A_CASES)
    assert any(kt == 2 and s == 1 for kt, _, _, _, s in TC.A_CASES)            # the whole time tap is padding
    assert {b for *_, b, _ in TC.A_CASES} == {1, 2, 3} == {s for *_, s in TC.A_CASES}
    old = TC.instantiations(OLD)
    missed = TC.ALL_KERNELS - {(k, n) for k, n, _ in old}
    assert missed == {(k, n) for k in ("forward", "dgrad", "wgrad") for n in (16, 24, 48, 56)}
    assert {nks for _, _, nks in old if nks} == {1, 4, 5, 8}
    assert not any(cin > cout for _, (cin, cout), *_ in OLD)


def test_grid_list_covers_every_tile_class():
    xs, ys = {x for x, _ in TC.B_GRIDS}, {y for _, y in TC.B_GRIDS}
    assert xs == set(TC.B_X) and ys == set(TC.B_Y)
    assert {1, 8, 9, 16, 17} <= xs and {16, 20, 32, 36} <= ys                  # one exact tile / run, one row / one float4 past it
    assert {y % 16 for y in ys} == {0, 4, 8, 12} and {y % 32 for y in ys} == set(range(0, 32, 4))
    assert all(sum(1 for g in TC.B_GRIDS if g[1] == y) == 2 for y in ys)
    assert all(sum(1 for g in TC.B_GRIDS if g[0] == x) >= 2 for x in xs)
    assert {(x % 8, y % 16) for x, y in TC.B_GRIDS} == {(a, c) for a in {x % 8 for x in xs} for c in (0, 4, 8, 12)}


def test_aggregation_cases_reach_every_launch_and_the_old_list_does_not():
    from tests.test_temporal_tail_gpu import AGG as OLD
    got = TC.aggregation_launch_set(TC.AGG_CASES)
    assert got == TC.ALL_AGG_LAUNCHES
    kernels = {k[:2] for k in got}
    assert {("aggregation", 1), ("aggregation", 2), ("dgrad", 1), ("dgrad", 2)} <= kernels
    assert {("forward", nch) for nch in (1, 2, 3, 4)} | {("wgrad", 1), ("wgrad", 2)} <= kernels
    assert {k[2] for k in got if k[0] == "wgrad"} == {128, 256, 384, 512}
    # the ring depths: NCHK = 1 runs 4 / 3 / 2 stages, NCHK = 2 runs 4 / 2 / 1; one stage only for N > 64 with Npad32 >= 224
    for kind in ("aggregation", "dgrad"):
        assert {k[2] for k in got if k[:2] == (kind, 1)} == {4, 3, 2}
        assert {k[2] for k in got if k[:2] == (kind, 2)} == {4, 2, 1}
    for n in range(1, 129):
        for npad in range(8, 257, 8):
            one_stage = TC.aggregation_launches(n, (npad,), 1)[0][2] == 1
            assert one_stage == (n > 64 and (npad + 31) // 32 * 32 >= 224), (n, npad)
    ns = {n for n, *_ in TC.AGG_CASES}
    assert {1, 7, 8, 9, 31, 32, 33, 63, 64, 65, 96, 127, 128} <= ns
    assert {len(p) for _, p, *_ in TC.AGG_CASES} == {1, 2, 3, 4}
    assert any(c % 8 for _, p, *_ in TC.AGG_CASES for c in p) and any(c % 8 == 0 for _, p, *_ in TC.AGG_CASES for c in p)
    npads = {sum(TC.round8(c) for c in p) for _, p, *_ in TC.AGG_CASES}
    assert {(v - 1) // 64 for v in npads} == {0, 1, 2, 3} and 256 in npads
    assert {r for _, _, r, *_ in TC.AGG_CASES} >= {0, 1, 23} and max(r for _, _, r, *_ in TC.AGG_CASES) >= 128
    assert {b for *_, b, _ in TC.AGG_CASES} == {1, 2, 3} == {s for *_, s in TC.AGG_CASES}
    old = TC.aggregation_launch_set([(n, p, r) for p, r, n in OLD.values()])
    assert {k[:2] for k in old if k[0] in ("aggregation", "dgrad")} == {("aggregation", 1)}


def test_aggregation_maps_cover_every_tile_class():
    pixels = {X * Y for _, _, _, (X, Y), _, _ in TC.AGG_CASES}
    assert pixels == set(TC.AGG_GRIDS) and all(p % 4 == 0 for p in pixels)
    assert all(X * Y == p for p, (X, Y) in TC.AGG_GRIDS.items())
    for tile in (64, 128):                                      # the backward / aggregation tile and the forward's
        assert {p % tile for p in pixels} >= {0, 4, tile - 4}, tile
        assert tile in pixels and tile + 4 in pixels and tile - 4 in pixels
    assert {4, 60} <= pixels and max(pixels) == 40000


@pytest.mark.parametrize("n,paths,r,grid,b,s", TC.AGG_CASES[::4], ids=lambda v: str(v).replace(" ", ""))
def test_aggregation_workspace_is_the_swapped_entry_rule(n, paths, r, grid, b, s):
    from fiery_b200.temporal import backward_weight_workspace_bytes
    X, Y = grid
    assert backward_weight_workspace_bytes((b, n, s, X, Y), paths, 0) == TC.entry_workspace_bytes(b, s, X * Y, n, paths, 0)


SUM_PIXELS = [1, 3, 4, 5, 255, 1023, 1024, 1025, 4095, 4096, 4097, 8193, 40000]


@pytest.mark.parametrize("pixels", SUM_PIXELS)
def test_spatial_sums_model_against_fp64(pixels):
    gen = np.random.default_rng(pixels)
    x = (gen.standard_normal((64, pixels)) * np.exp2(gen.integers(-4, 5, (64, pixels)))).astype(np.float32)
    got = TC.spatial_sums_model(x, pixels)
    assert got.dtype == np.float32 and got.shape == (64,)
    ref = x.astype(np.float64).sum(1)
    bound = 4 * math.sqrt(pixels) * np.spacing(np.abs(x).max(1).astype(np.float32)).astype(np.float64)
    assert np.all(np.abs(got.astype(np.float64) - ref) <= bound), float(np.max(np.abs(got - ref) / bound))
    ints = gen.integers(-3, 4, (2, 3, pixels)).astype(np.float32)
    assert np.array_equal(TC.spatial_sums_model(ints, pixels), ints.astype(np.float64).sum(-1))


def _with(pixels, values):
    x = np.zeros(pixels, np.float32)
    for i, v in values.items():
        x[i] = v
    return float(TC.spatial_sums_model(x, pixels))


def test_spatial_sums_model_order_on_chosen_values():
    """2^24 and two 1.0s: 2^24 + 1 rounds back to 2^24 (ties to even) but 2^24 + 2 is exact, so where the two 1.0s meet each other
    before meeting 2^24 shows the order."""
    big, pixels = 2.0 ** 24, 4 * 512 + 8               # thread 0 takes chunks 0, 256 and 512, thread 1 chunks 1, 257 and 513, ...
    assert _with(pixels, {0: big, 1024: 1.0, 2048: 1.0}) == big          # one lane accumulator, in chunk order
    assert _with(pixels, {0: big, 2: 1.0, 3: 1.0}) == big + 2            # lanes 2 and 3 are added before lanes 0 and 1
    assert _with(pixels, {0: big, 1: 1.0, 2: 1.0}) == big                # lanes 0 and 1 first
    assert _with(pixels, {0: big, 4: 1.0, 68: 1.0}) == big + 2           # threads 1 and 17 meet at butterfly offset 16
    assert _with(pixels, {0: big, 4: 1.0, 8: 1.0}) == big                # threads 1 and 2 meet thread 0 first
    assert _with(pixels, {0: big, 128: 1.0, 256: 1.0}) == big            # warps 0, 1, 2: added one after the other


def _cc_desc(b, s, X, Y, cin, cout, kt):
    d = _lib.CausalConv3dDesc()
    d.batch, d.frames, d.grid_x, d.grid_y, d.in_channels, d.out_channels, d.kt = b, s, X, Y, cin, cout, kt
    return d


@pytest.mark.parametrize("tiles", TC.D_TILE_COUNTS)
def test_chunk_edge_shapes_have_the_tile_counts_they_are_named_for(tiles):
    from fiery_b200.temporal import backward_weight_workspace_bytes
    lib = _lib.load()
    b, s, X, Y = TC.D_CAUSAL[tiles]
    assert TC.causal_wgrad_tiles(b, s, X, Y) == tiles
    for cin, cout, kt in ((9, 17, 2), (35, 35, 1)):
        assert lib.fiery_causal_conv3d_backward_weight_workspace_bytes(_cc_desc(b, s, X, Y, cin, cout, kt)) == \
            TC.causal_workspace_bytes(b, s, X, Y, cin, cout, kt)
    b, s, (X, Y) = TC.D_ENTRY[tiles]
    assert TC.entry_wgrad_tiles(b, s, X * Y) == tiles
    for K, segs, E in BLOCKS.values():
        assert backward_weight_workspace_bytes((b, K, s, X, Y), segs, E) == TC.entry_workspace_bytes(b, s, X * Y, K, segs, E)
    bounds = TC.chunk_bounds(tiles)
    assert bounds[0][0] == 0 and bounds[-1][1] == tiles and all(a[1] == b_[0] for a, b_ in zip(bounds, bounds[1:]))
    sizes = {t1 - t0 for t0, t1 in bounds}
    assert min(sizes) >= 1 and (len(sizes) == 2) == (tiles > 128 and tiles % 128 != 0)


def _f(bits):
    return struct.unpack("<f", struct.pack("<I", bits))[0]


@pytest.mark.parametrize("bits,rna,trunc", [
    (0x3F801000, 0x3F802000, 0x3F800000),      # tie: away from zero
    (0x3F800FFF, 0x3F800000, 0x3F800000),      # just below the tie
    (0x3F801001, 0x3F802000, 0x3F800000),      # just above
    (0x3FFFFFFF, 0x40000000, 0x3FFFE000),      # mantissa all ones: the carry goes into the exponent
    (0xBF801000, 0xBF802000, 0xBF800000),      # negative tie: away from zero
    (0xBFFFF000, 0xC0000000, 0xBFFFE000),
    (0x00000000, 0x00000000, 0x00000000),
    (0x80000000, 0x80000000, 0x80000000),
    (0x00001000, 0x00002000, 0x00000000),      # denormal: stays finite
    (0x40490FDB, 0x40490000, 0x40490000),      # pi: below half
    (0x402DF854, 0x402E0000, 0x402DE000),      # e: above half
])
def test_tf32_rounding_on_bit_patterns(bits, rna, trunc):
    t = torch.tensor([_f(bits)], dtype=torch.float32)
    got_r, got_t = TC.tf32_rna(t), TC.tf32_trunc(t)
    assert got_r.view(torch.int32).item() & 0xFFFFFFFF == rna and got_t.view(torch.int32).item() & 0xFFFFFFFF == trunc
    assert bool(torch.isfinite(got_r).all()) and bool(torch.isfinite(got_t).all())
    assert abs(got_r.double().item() - t.double().item()) <= abs(got_t.double().item() - t.double().item())


def test_full_mantissa_values_tell_the_roundings_apart():
    v = TC.full_mantissa((3, 5, 7, 11), seed=0)
    r, t = TC.tf32_rna(v), TC.tf32_trunc(v)
    assert bool(torch.isfinite(v).all()) and float(v.abs().max()) < 1e3
    assert float((r != t).float().mean()) > 0.4 and float((r == t).float().mean()) > 0.2
    up, down = (r.double() - v.double()) > 0, (r.double() - v.double()) < 0
    assert bool(up.any()) and bool(down.any())                                 # rna errs on both sides, truncation only towards zero
    assert bool(((t.double() - v.double()) * v.double().sign() <= 0).all())
    low = v.view(torch.int32) & 0x1FFF
    assert all(int((low == k).sum()) > 50 for k in (0x1000, 0x0FFF, 0x1FFF))


def _conv_reference(x, w, gy):
    kt = w.shape[2]
    xd = x.double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    y = F.conv3d(F.pad(xd, (1, 1, 1, 1, kt - 1, 0)), wd)
    y.backward(gy.double())
    return y.detach(), xd.grad, wd.grad


@pytest.mark.parametrize("kt", [1, 2])
@pytest.mark.parametrize("c_out,c_in", [(17, 17), (35, 35), (24, 9), (5, 12)])
def test_permutation_expectations_equal_fp64_conv(kt, c_out, c_in):
    w, where = TC.permutation_weight(c_out, c_in, kt, seed=c_out + kt)
    gen = torch.Generator().manual_seed(1)
    x = torch.randn((2, c_in, 3, 5, 8), generator=gen)
    gy = torch.randn((2, c_out, 3, 5, 8), generator=gen)
    y, gx, _ = _conv_reference(x, w, gy)
    assert torch.equal(TC.shifted_forward(x, where, kt).double(), y)
    if c_out <= c_in:                                                          # no input channel used twice
        assert torch.equal(TC.shifted_backward(gy, where, kt, c_in).double(), gx)
    else:
        with pytest.raises(AssertionError, match="used twice"):
            TC.shifted_backward(gy, where, kt, c_in)


@pytest.mark.parametrize("kt", [1, 2])
def test_one_hot_expectations_equal_fp64_conv(kt):
    c_in, c_out, b, s, X, Y = 7, 10, 2, 3, 4, 8
    gen = torch.Generator().manual_seed(2)
    x = torch.randn((b, c_in, s, X, Y), generator=gen)
    gy = torch.randn((b, c_out, s, X, Y), generator=gen)
    w = torch.zeros(c_out, c_in, kt, 3, 3)
    pos_o = TC.one_hot_positions(c_out, b, s, X, Y, seed=3)
    assert pos_o[:4, 2:].tolist() == [[0, 0], [0, Y - 1], [X - 1, 0], [X - 1, Y - 1]]
    assert torch.equal(TC.taps_of_x(x, pos_o, kt).double(), _conv_reference(x, w, TC.one_hot(pos_o, b, s, X, Y))[2])
    pos_i = TC.one_hot_positions(c_in, b, s, X, Y, seed=4)
    assert torch.equal(TC.taps_of_grad(gy, pos_i, kt).double(), _conv_reference(TC.one_hot(pos_i, b, s, X, Y), w, gy)[2])


@pytest.mark.parametrize("kt", [1, 2])
@pytest.mark.parametrize("c_out,c_in", [(17, 17), (9, 35), (64, 3)])
def test_weights_read_back_through_one_hot_maps(kt, c_out, c_in):
    w = torch.randn((c_out, c_in, kt, 3, 3), generator=torch.Generator().manual_seed(5))
    x = TC.cell_one_hot(c_in, kt, 0)
    gy = TC.cell_one_hot(c_out, kt, kt - 1)
    assert x.shape[-1] % 4 == 0 and gy.shape[-1] % 4 == 0
    y = F.conv3d(F.pad(x.double(), (1, 1, 1, 1, kt - 1, 0)), w.double())
    assert torch.equal(TC.weights_as_output(w).double(), y)
    assert int((y != 0).sum()) == w.numel()                                    # every weight is one output element
    xd = torch.zeros((1, c_in, kt, *gy.shape[-2:]), dtype=torch.float64, requires_grad=True)
    F.conv3d(F.pad(xd, (1, 1, 1, 1, kt - 1, 0)), w.double()).backward(gy.double())
    assert torch.equal(TC.weights_as_input_gradient(w).double(), xd.grad)


def test_guarded_and_poisoned_buffers():
    buf, view = TC.guarded(10, 5, 7, "cpu")
    assert view.data_ptr() % 16 == 0 and bool(view.isnan().all()) and buf.numel() >= 22
    with pytest.raises(AssertionError, match="never written"):
        TC.assert_written_and_contained(buf, view, "out")
    view.zero_()
    TC.assert_written_and_contained(buf, view, "out")
    for at in (0, 7, 18, buf.numel() - 1):                                     # in front of the view and behind it
        b2, v2 = TC.guarded(10, 5, 7, "cpu")
        v2.zero_()
        b2[at] = 1.0
        with pytest.raises(AssertionError, match="outside"):
            TC.assert_written_and_contained(b2, v2, "out")
    x = torch.arange(2 * 3 * 2 * 2 * 4, dtype=torch.float32).view(2, 3, 2, 2, 4)
    p = TC.poisoned(x, "cpu")
    assert p.is_contiguous() and torch.equal(p, x)
    assert bool(p.as_strided((8,), (1,), p.storage_offset() - 8).isnan().all())
    assert bool(p.as_strided((8,), (1,), p.storage_offset() + p.numel()).isnan().all())
    q = TC.poisoned_frame_major(x, "cpu", gap=4)
    assert torch.equal(q, x) and q.stride() == (2 * 7 * 8, 8, 7 * 8, 4, 1)
    assert bool(q.as_strided((4 * 8,), (1,), q.storage_offset() + 3 * 8).isnan().all())      # the gap after frame 0's channels
    # a strided guarded view: the gaps count as outside
    buf = torch.full((q.numel() * 4,), TC.SENTINEL)
    gx = buf.as_strided(q.size(), q.stride(), 16)
    gx.fill_(0.0)
    TC.assert_written_and_contained(buf, gx, "gx")
    buf[16 + 3 * 8] = 0.0
    with pytest.raises(AssertionError, match="outside"):
        TC.assert_written_and_contained(buf, gx, "gx")
