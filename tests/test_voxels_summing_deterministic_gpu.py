"""GPU: VoxelsSumming's deterministic forward (fiery_voxels_summing_forward_deterministic, selected by
torch.use_deterministic_algorithms(True)).  Runs that cross the edge of a 64-row chunk are summed per chunk and their pieces added in
chunk order instead of atomically: three calls must be bit-equal, every sum within the fp32 bound of a sequential sum against fp64,
and the kept coordinates and the backward unchanged."""
import pytest
import torch

from fiery_b200.geometry import VoxelsSumming

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -24
CHUNK = 64


def _ranks(n, lengths):
    """Ascending ranks of n rows: runs of the given lengths first (cycling), the rest single rows."""
    seg = torch.empty(n, dtype=torch.int64)
    r, s, i = 0, 0, 0
    while r < n:
        ln = lengths[i % len(lengths)] if lengths else 1
        seg[r:r + ln] = s
        r, s, i = r + ln, s + 1, i + 1
    return (seg * 5 + 2).to(DEV)


def _run(x, ranks, deterministic):
    geometry = torch.stack([ranks, torch.arange(ranks.numel(), device=DEV), ranks % 3], 1)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        xr = x.detach().requires_grad_(True)
        sums, kept = VoxelsSumming.apply(xr, geometry, ranks)
        g = torch.linspace(-1.0, 1.0, sums.numel(), device=DEV).view_as(sums)
        (sums * g).sum().backward()
    finally:
        torch.use_deterministic_algorithms(old)
    return sums.detach(), kept, xr.grad


def _check(x, ranks):
    runs = [_run(x, ranks, True) for _ in range(3)]
    for s, k, g in runs[1:]:
        assert torch.equal(s.view(torch.int32), runs[0][0].view(torch.int32))
        assert torch.equal(k, runs[0][1]) and torch.equal(g, runs[0][2])
    s_def, k_def, g_def = _run(x, ranks, False)
    s, k, g = runs[0]
    assert torch.equal(k, k_def) and torch.equal(g, g_def)             # coordinates and backward as before
    # fp64 reference and the bound of a sequential fp32 sum: |err| <= (len - 1) * u * sum |x| (+ one rounding of the result)
    _, seg, counts = torch.unique_consecutive(ranks, return_inverse=True, return_counts=True)
    xd = x.double().cpu()
    seg = seg.cpu()
    exact = torch.zeros(int(counts.numel()), x.shape[1], dtype=torch.float64).index_add_(0, seg, xd)
    absum = torch.zeros_like(exact).index_add_(0, seg, xd.abs())
    bound = (counts.cpu().double()[:, None] + 1) * U * absum + 1e-30
    assert bool(((s.double().cpu() - exact).abs() <= bound).all())
    return s


@pytest.mark.parametrize("lengths", [[130], [200, 70], [150, 3, 256, 1], [CHUNK * 37 + 5]], ids=["3chunks", "4chunks", "mixed", "many"])
@pytest.mark.parametrize("C", [1, 64, 1024])
def test_runs_across_chunks(lengths, C):
    n = 20000 if C < 1024 else 4000
    x = torch.randn(n, C, generator=torch.Generator(device=DEV).manual_seed(C + len(lengths)), device=DEV)
    _check(x, _ranks(n, lengths))


def test_all_rows_one_voxel():
    n = 4_200_000
    x = torch.randn(n, 4, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
    s = _check(x, torch.full((n,), 9, dtype=torch.int64, device=DEV))
    assert s.shape == (1, 4)


def test_row_stride():
    n, C = 9000, 48
    base = torch.randn(n, 80, generator=torch.Generator(device=DEV).manual_seed(4), device=DEV)
    x = base[:, 16:16 + C]
    assert x.stride(0) == 80
    _check(x, _ranks(n, [300, 65, 64, 63]))
