"""GPU: VoxelsSumming (fiery_b200/csrc/voxels_summing.cu) across the shapes its C ABI accepts.

  A. Row counts at the edges of the 64-row chunks of the forward, the 2048-row tiles of the plan's scan, and the rounds of 1024 tiles
     that vs_scan_tiles_kernel carries a running total across (2048 * 1024 rows and more); runs that end exactly on chunk and tile
     edges, one run across every chunk of a multi-million-row input, all singletons and random runs.
  B. Channel counts from 1 to 1024: every block shape vs_forward picks (C < 3, C not a multiple of 32, one row of 256..1024 threads);
     1025 is rejected.
  C. The host layer: fp16 / bf16 features, int32 ranks and geometry, a row stride larger than C.

Small-integer features make every sum exact in fp32, whatever order the atomics add in: sums, kept coordinates and gradients must then
be bit-exact against int64 / fp64 references.  Random fp32 features are compared with oracle.direct_segment_sum in fp64 at a bar from
the run length.  Through the C ABI, sums_out / coords_out / grad_feats start as NaN / -1 and are followed by a sentinel margin: all U
rows must be written and nothing past them."""
import ctypes

import pytest
import torch

from fiery_b200 import _lib
from fiery_b200.geometry import VoxelsSumming
from oracle import lift_oracle as O

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
U = 2.0 ** -24
SENTINEL = -1.0e30
COORD_SENTINEL = -7777
MARGIN_ROWS = 64
CHUNK, TILE, ROUND = 64, 2048, 2048 * 1024       # forward chunk, scan tile, rows per round of vs_scan_tiles_kernel


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ranks(n, pattern, seed):
    """Ascending int64 ranks of n rows whose runs follow `pattern`."""
    r = torch.arange(n, device=DEV)
    if pattern == "singletons":
        start = torch.ones(n, dtype=torch.bool, device=DEV)
    elif pattern == "one":
        start = r == 0
    elif pattern == "edges":
        # runs start on every chunk edge, so they end exactly on one; around the tile edges also runs of a single row
        start = (r % CHUNK == 0) | (r % TILE == 1) | (r % TILE == TILE - 1)
    else:                                                                # random runs of 1..150 rows, many straddling a chunk
        start = torch.rand(n, generator=_gen(seed), device=DEV) < 1.0 / 75
    start[:1] = True
    return (torch.cumsum(start.long(), 0) - 1) * 3 + 11


def _segments(ranks):
    n = ranks.numel()
    start = torch.ones(n, dtype=torch.bool, device=DEV)
    start[1:] = ranks[1:] != ranks[:-1]
    seg = torch.cumsum(start.long(), 0) - 1
    last = torch.ones(n, dtype=torch.bool, device=DEV)
    last[:-1] = start[1:]
    return seg, last


def _coords(ranks):
    """Per-row coordinates that differ within a run, so the kept row (the last of its run) is checked."""
    n = ranks.numel()
    r = torch.arange(n, device=DEV)
    return torch.stack([ranks, r, r % 7 + 1], 1).contiguous()                # never -1, the unwritten marker


def _vs_abi(feats, coords, ranks, stride=None):
    """Plan, forward and backward through the C ABI.  feats (n, C) float32 with row stride `stride` (default its own).  The outputs go
    into guarded buffers (NaN / -1, then MARGIN_ROWS rows of sentinels); returns (sums (U, C), kept (U, 3), seg (n,) int32)."""
    lib = _lib.load()
    n, C = feats.shape
    seg = torch.empty(max(n, 1), dtype=torch.int32, device=DEV)
    n_seg = ctypes.c_int64(-1)
    _lib.check(lib.fiery_voxels_summing_plan(n, ranks.data_ptr(), seg.data_ptr(), ctypes.byref(n_seg), _stream()),
               "fiery_voxels_summing_plan")
    Useg = int(n_seg.value)
    sums = torch.full(((Useg + MARGIN_ROWS) * C,), float("nan"), device=DEV)
    sums[Useg * C:] = SENTINEL
    kept = torch.full(((Useg + MARGIN_ROWS) * 3,), -1, dtype=torch.int64, device=DEV)
    kept[Useg * 3:] = COORD_SENTINEL
    _lib.check(lib.fiery_voxels_summing_forward(n, C, feats.stride(0) if stride is None else stride, feats.data_ptr(),
                                                coords.data_ptr(), seg.data_ptr(), Useg, sums.data_ptr(), kept.data_ptr(),
                                                _stream()), "fiery_voxels_summing_forward")
    assert not bool(sums[:Useg * C].isnan().any()), "sums never written"
    assert bool((sums[Useg * C:] == SENTINEL).all()), "store past the sums"
    assert not bool((kept[:Useg * 3] == -1).any()), "kept coordinates never written"
    assert bool((kept[Useg * 3:] == COORD_SENTINEL).all()), "store past the kept coordinates"
    return sums[:Useg * C].view(Useg, C), kept[:Useg * 3].view(Useg, 3), seg[:n]


def _vs_backward_abi(gsums, seg, n, C):
    lib = _lib.load()
    buf = torch.full(((n + MARGIN_ROWS) * C,), float("nan"), device=DEV)
    buf[n * C:] = SENTINEL
    _lib.check(lib.fiery_voxels_summing_backward(n, C, gsums.data_ptr(), seg.data_ptr(), buf.data_ptr(), _stream()),
               "fiery_voxels_summing_backward")
    assert not bool(buf[:n * C].isnan().any()), "gradient never written"
    assert bool((buf[n * C:] == SENTINEL).all()), "store past the gradient"
    return buf[:n * C].view(n, C)


def _check_exact(feats, ranks, stride=None, dense=None):
    """Small-integer features: sums, kept coordinates, segment ids and gradients bit-exact.  Every partial sum is an integer of
    magnitude at most 2 * n_rows < 2^24, so fp32 adds them exactly in any order."""
    n, C = feats.shape
    coords = _coords(ranks)
    sums, kept, seg = _vs_abi(feats, coords, ranks, stride)
    want_seg, last = _segments(ranks)
    Uw = int(want_seg[-1]) + 1 if n else 0
    assert sums.shape == (Uw, C)
    vals = feats if dense is None else dense
    want = torch.zeros(Uw, C, dtype=torch.float64, device=DEV).index_add_(0, want_seg, vals.double())
    assert torch.equal(sums.double(), want)
    assert torch.equal(kept, coords[last])
    assert torch.equal(seg.long(), want_seg)
    gsums = torch.randint(-9, 10, (Uw, C), generator=_gen(n + C), device=DEV).float()
    assert torch.equal(_vs_backward_abi(gsums, seg, n, C), gsums[want_seg])


def _int_feats(n, C, seed):
    return torch.randint(-2, 3, (n, C), generator=_gen(seed), device=DEV).float()


ROWS = [1, CHUNK - 1, CHUNK, CHUNK + 1, TILE - 1, TILE, TILE + 1, ROUND - 1, ROUND + 1, 2 * ROUND + 5]
PATTERNS = ["random", "edges", "one", "singletons"]


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("n", ROWS)
def test_row_counts_and_runs_are_exact(n, pattern):
    C = 2 if n > ROUND // 2 else 5
    ranks = _ranks(n, pattern, seed=n)
    _check_exact(_int_feats(n, C, seed=n + len(pattern)), ranks)


def test_zero_rows():
    lib = _lib.load()
    n_seg = ctypes.c_int64(-1)
    _lib.check(lib.fiery_voxels_summing_plan(0, None, None, ctypes.byref(n_seg), _stream()), "plan, 0 rows")
    assert n_seg.value == 0
    _lib.check(lib.fiery_voxels_summing_forward(0, 4, 4, None, None, None, 0, None, None, _stream()), "forward, 0 rows")
    _lib.check(lib.fiery_voxels_summing_backward(0, 4, None, None, None, _stream()), "backward, 0 rows")
    x = torch.zeros(0, 4, device=DEV, requires_grad=True)
    sums, kept = VoxelsSumming.apply(x, torch.zeros(0, 3, dtype=torch.long, device=DEV), torch.zeros(0, dtype=torch.long, device=DEV))
    assert sums.shape == (0, 4) and kept.shape == (0, 3)


CHANNELS = [1, 2, 3, 4, 31, 32, 33, 100, 255, 256, 257, 1024]


@pytest.mark.parametrize("C", CHANNELS)
def test_channel_counts(C):
    """Every block shape of vs_forward: tx = C rounded up to 32 (at least 32), ty = 256 / tx rows of chunks, one row from 256 on.
    Integers bit-exact; random fp32 against the fp64 direct sum, element-wise: a run of L rows is added in at most L - 1 fp32 additions
    (in the chunk and by the atomics between chunks), so |sum - exact| <= (L - 1) u sum |x| (to first order; the bar takes L u)."""
    n = 5 * TILE + 17
    ranks = _ranks(n, "random", seed=C)
    _check_exact(_int_feats(n, C, seed=C), ranks)
    feats = torch.randn(n, C, generator=_gen(C + 1), device=DEV)
    sums, _, _ = _vs_abi(feats, _coords(ranks), ranks)
    exact = O.direct_segment_sum(feats.cpu(), ranks.cpu())
    seg, _ = _segments(ranks)
    L = torch.bincount(seg).double().cpu()
    abs_sum = O.direct_segment_sum(feats.abs().cpu(), ranks.cpu())
    bar = L.view(-1, 1) * U * abs_sum
    err = (sums.cpu().double() - exact).abs()
    assert bool((err <= bar).all()), float((err - bar).max())
    assert int(L.max()) > CHUNK                                           # some runs cross a chunk edge


@pytest.mark.parametrize("C,stride", [(1025, 1025), (0, 4), (8, 7), (-1, 4)])
def test_bad_shapes_are_rejected(C, stride):
    lib = _lib.load()
    buf = torch.zeros(64, device=DEV)
    seg = torch.zeros(4, dtype=torch.int32, device=DEV)
    rc = lib.fiery_voxels_summing_forward(4, C, stride, buf.data_ptr(), buf.data_ptr(), seg.data_ptr(), 1, buf.data_ptr(),
                                          buf.data_ptr(), _stream())
    assert rc != 0 and lib.fiery_last_error()
    n_seg = ctypes.c_int64(0)
    assert lib.fiery_voxels_summing_plan(1 << 31, buf.data_ptr(), seg.data_ptr(), ctypes.byref(n_seg), _stream()) != 0
    assert lib.fiery_voxels_summing_plan(-1, buf.data_ptr(), seg.data_ptr(), ctypes.byref(n_seg), _stream()) != 0


def test_row_stride_larger_than_channels_abi():
    """Rows C = 33 wide at a stride of 40, NaN in the 7 columns between: never read."""
    n, C, S = 3 * TILE + 5, 33, 40
    ranks = _ranks(n, "random", seed=3)
    dense = _int_feats(n, C, seed=3)
    buf = torch.full((n, S), float("nan"), device=DEV)
    buf[:, :C] = dense
    _check_exact(buf[:, :C], ranks, stride=S, dense=dense)


# ==== host layer ===============================================================================================================
def _host_case(n, C, seed):
    """Small-integer features: the sums are exact, so two calls agree bit for bit whatever order the atomics add in."""
    ranks = _ranks(n, "random", seed)
    return _int_feats(n, C, seed), _coords(ranks), ranks


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_host_half_precision_features(dtype):
    """Result and gradient in the features' dtype, equal to the fp32 path on the widened features, rounded."""
    feats, coords, ranks = _host_case(3000, 64, seed=5)
    x16 = feats.to(dtype).requires_grad_(True)
    sums, kept = VoxelsSumming.apply(x16, coords, ranks)
    assert sums.dtype == dtype and kept.dtype == torch.int64
    x32 = x16.detach().float().requires_grad_(True)
    sums32, kept32 = VoxelsSumming.apply(x32, coords, ranks)
    assert torch.equal(sums.detach(), sums32.detach().to(dtype)) and torch.equal(kept, kept32)
    gout = torch.randn(sums.shape, generator=_gen(6), device=DEV).to(dtype)
    sums.backward(gout)
    sums32.backward(gout.float())
    assert x16.grad.dtype == dtype
    assert torch.equal(x16.grad, x32.grad.to(dtype))


def test_host_int32_ranks_and_geometry():
    feats, coords, ranks = _host_case(4000, 16, seed=7)
    a, ka = VoxelsSumming.apply(feats, coords.int(), ranks.int())
    b, kb = VoxelsSumming.apply(feats, coords, ranks)
    assert ka.dtype == torch.int32
    assert torch.equal(a, b) and torch.equal(ka.long(), kb)


def test_host_row_stride_larger_than_channels():
    """A (n, C) view of a wider NaN-padded tensor goes in without a copy; the NaN columns are never read, and the gradient lands in
    the view's shape."""
    n, C = 2 * TILE + 9, 20
    feats, coords, ranks = _host_case(n, C, seed=9)
    wide = torch.full((n, C + 12), float("nan"), device=DEV)
    wide[:, 3:3 + C] = feats
    view = wide[:, 3:3 + C].detach().requires_grad_(True)
    assert view.stride() == (C + 12, 1)
    got, _ = VoxelsSumming.apply(view, coords, ranks)
    x = feats.clone().requires_grad_(True)
    want, _ = VoxelsSumming.apply(x, coords, ranks)
    assert torch.equal(got, want)
    gout = torch.randn(want.shape, generator=_gen(10), device=DEV)
    got.backward(gout)
    want.backward(gout)
    assert torch.equal(view.grad, x.grad)
