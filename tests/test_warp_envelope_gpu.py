"""GPU: the BEV warp (fiery_b200/csrc/warp.cu, warp_sample.cuh) across the shapes its C ABI accepts, against fp64.

  A. Forward and backward over map shapes from 1 x 1 to 400 x 200: both 8-channel (forward) and 32-channel (backward) blocks with full
     and partial tails, the generic kernels and the <40000> / <80000> instances (the reference's 200 x 200 and 400 x 200 grids),
     identity, random rotations and translations that push most of the map out of range; bilinear and nearest.
  B. Exact cases: power-of-two maps, small-integer features and dyadic maps (quarter turns, integer and half-pixel shifts), where
     every sample position and weight is exact, so the kernels must agree with fp64 bit for bit; the half-pixel nearest cases pin
     grid_sample's round-half-to-even tie rule.
  C. The gather adjoint as the exact transpose of the forward, every source pixel of the 200 x 200 and 400 x 200 maps probed: a
     candidate missing from an adjoint window shows however small its weight.
  D. Layout and contract through the C ABI: map strides, NaN gaps that must never be read, copy masks, n_maps = 0, rejected shapes.
  E. Pose algebra (fiery_warp_theta) against the fp64 oracle.
  F. The host layer (warp_features / cumulative_warp_features): dtypes and strided, expanded and channels-last inputs.
  G. One 11264 x 11264 map with 18 channels: channel offsets past 2^31 elements in the backward.

Kernel outputs go into a NaN-filled buffer whose gaps between maps and margin after the last map hold a sentinel: every output must
be written and nothing else may change.  The fp64 reference is torch's grid_sample in float64 on a grid computed in float64 from the
kernel's own fp32 theta."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fiery_b200 import _lib
from fiery_b200.warp import _device_theta, cumulative_warp_features, warp_features
from oracle import warp_oracle as WO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SENTINEL = -1.0e30                  # a value no warp output here can take
U = 2.0 ** -24                      # unit roundoff of fp32
EXT = 50.0                          # spatial extent of the random maps (only the ratio translation / extent matters)


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device=DEV).float()


# ==== helpers ======================================================================================================================
def _warp(forward, src, theta, nearest, mask=None, src_stride=None, out_stride=None):
    """One fiery_warp_features_forward / _backward call.  src (n, C, H, W) has dense channel planes; its map stride is src_stride
    (default src.stride(0)).  The output goes into a buffer of map stride out_stride (default C*H*W) whose outputs start as NaN and
    whose gaps and margin hold SENTINEL.  The margin covers every store a block can address past the last map: 32 channel planes
    (the backward's channel block) and one thread block of pixels.  Returns the outputs as (n, C, H, W)."""
    n, C, H, W = src.shape
    chw = C * H * W
    ost = chw if out_stride is None else out_stride
    total = (n - 1) * ost + chw + 32 * H * W + 256
    buf = torch.full((total,), SENTINEL, device=DEV)
    outs = buf.as_strided((n, chw), (ost, 1))
    outs.fill_(float("nan"))
    fn = _lib.load().fiery_warp_features_forward if forward else _lib.load().fiery_warp_features_backward
    _lib.check(fn(n, C, H, W, src.data_ptr(), src.stride(0) if src_stride is None else src_stride, theta.data_ptr(),
                  mask.data_ptr() if mask is not None else None, buf.data_ptr(), ost, nearest, _stream()),
               "fiery_warp_features_" + ("forward" if forward else "backward"))
    assert not bool(outs.isnan().any()), ("outputs never written", int(outs.isnan().sum()))
    rest = buf.clone()
    rest.as_strided((n, chw), (ost, 1)).fill_(SENTINEL)
    assert bool((rest == SENTINEL).all()), "store outside the outputs"
    return outs.view(n, C, H, W)


def _grid64(theta, H, W):
    """affine_grid (align_corners=False) in float64 on the given (fp32) theta: centres x_i = (2i+1)/W - 1, grid = theta @ (x, y, 1)."""
    th = theta.double().view(-1, 2, 3)
    xs = (2.0 * torch.arange(W, dtype=torch.float64, device=DEV) + 1.0) / W - 1.0
    ys = (2.0 * torch.arange(H, dtype=torch.float64, device=DEV) + 1.0) / H - 1.0
    X, Y = xs.view(1, 1, W), ys.view(1, H, 1)
    gx = th[:, 0, 0, None, None] * X + th[:, 0, 1, None, None] * Y + th[:, 0, 2, None, None]
    gy = th[:, 1, 0, None, None] * X + th[:, 1, 1, None, None] * Y + th[:, 1, 2, None, None]
    return torch.stack([gx, gy], -1)


def _ref64(x, theta, nearest):
    """grid_sample in float64 (zero padding, align_corners=False; nearest rounds half to even)."""
    _, _, H, W = x.shape
    return F.grid_sample(x.double(), _grid64(theta, H, W), mode="nearest" if nearest else "bilinear", padding_mode="zeros",
                         align_corners=False)


def _ref64_backward(g, theta, nearest):
    x = torch.zeros(g.shape, dtype=torch.float64, device=DEV, requires_grad=True)
    _ref64(x, theta, nearest).backward(g.double())
    return x.grad


def _pixel_coords64(theta, H, W):
    """The fp64 sample position (ix, iy) of every output pixel, in pixels (grid_sample's unnormalisation)."""
    grid = _grid64(theta, H, W)
    return ((grid[..., 0] + 1.0) * W - 1.0) / 2.0, ((grid[..., 1] + 1.0) * H - 1.0) / 2.0


def _coord_error(theta, H, W):
    """Bound on |ix_fp32 - ix_exact| and |iy_fp32 - iy_exact| per map, in pixels, for the kernel's sample_coords.

    With u = 2^-24 and G = |t0| + |t1| + |t2| (the x row of theta):
      x_i = fl(fl((2i+1) / W) - 1): the quotient is below 2 and the difference below 1 in magnitude, so |dx_i| <= 2u + u = 3u (same for y_j).
      gx = fma(t0, x_i, fma(t1, y_j, t2)): the input errors give (3|t0| + 3|t1|) u, the two roundings at most (|t1| + |t2|) u and G u:
           |dgx| <= 5 G u.
      ix = ((gx + 1) W - 1) / 2: the sum rounds by (G + 1) u, the product by (G + 1) W u, the difference by ((G + 1) W + 1) u, the
           halving is exact; with the propagated W |dgx|: |dix| <= (W (7G + 2) + (G + 1) W + 1) u / 2 <= W (4G + 2) u.
    Same for iy with H and the y row.  The fp64 reference's own error is below 2^-40 pixels here and is ignored."""
    th = theta.double().view(-1, 2, 3).abs().sum(-1)                    # (n, 2): G of each row
    return W * (4.0 * th[:, 0] + 2.0) * U, H * (4.0 * th[:, 1] + 2.0) * U


def _flows(rng, n, far):
    """(n, 6) flows of the kind write_theta turns into a map: any z rotation and an xy translation, |t| <= 0.8 of the extent, or
    (far) 1.1 to 1.9 of it along at least one axis, which leaves most of the map out of range."""
    f = np.zeros((n, 6), np.float32)
    f[:, 5] = rng.uniform(-np.pi, np.pi, n)
    t = rng.uniform(-0.8, 0.8, (n, 2))
    if far:
        axis = rng.integers(0, 2, n)
        t[np.arange(n), axis] = rng.uniform(1.1, 1.9, n) * rng.choice([-1.0, 1.0], n)
    f[:, :2] = t * EXT
    return f


def _rotation_thetas(seed, n_near, n_far):
    rng = np.random.default_rng(seed)
    flow = np.concatenate([_flows(rng, n_near, False), _flows(rng, n_far, True)])
    theta, _ = _device_theta(torch.from_numpy(flow).to(DEV), (EXT, EXT), cumulative=False)
    return theta                                                         # the GPU's own fp32 theta (write_theta)


IDENTITY = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0]


def _sweep_thetas(seed):
    """identity, two random rotations with moderate translations, one pushed mostly out of range"""
    eye = torch.tensor(IDENTITY, device=DEV).view(1, 2, 3)
    return torch.cat([eye, _rotation_thetas(seed, 2, 1)])


def _window_bound(H, W):
    """Most output pixels whose sample can touch one source pixel: the candidate window of adjoint_scan_begin, which the window model
    (tests/test_warp_window_model.py) bounds by 16 on square and 30 on rectangular maps."""
    return 16 if H == W else 30


# ==== A. sweep against fp64 ======================================================================================================
SMALL_SHAPES = [(1, 1), (1, 7), (7, 1), (3, 5), (13, 11), (64, 64)]
CHANNELS = [1, 7, 8, 9, 31, 32, 33, 64, 65]
# (H, W, C): the small maps with every channel count; the template instances (<40000>: 200 x 200, 160 x 250; <80000>: 400 x 200,
# 200 x 400, 320 x 250) and a generic plane just off 40000 (201 x 199) with C = 64, and a few partial tails on the large planes
SWEEP = ([(h, w, c) for h, w in SMALL_SHAPES for c in CHANNELS]
         + [(h, w, 64) for h, w in [(200, 200), (160, 250), (400, 200), (200, 400), (320, 250), (201, 199)]]
         + [(160, 250, 33), (320, 250, 65), (201, 199, 9)])


@pytest.mark.parametrize("nearest", [0, 1], ids=["bilinear", "nearest"])
@pytest.mark.parametrize("H,W,C", SWEEP)
def test_sweep_matches_fp64(H, W, C, nearest):
    """Forward and backward against fp64 grid_sample on the kernel's theta.

    Bilinear forward: out is Lipschitz in the sample position with constant 2 max|x| per axis (a weight moves between two neighbours),
    and the kernel's weights and four-term sum round by at most 8u max|x|: |out - ref| <= max|x| (2 (dx + dy) + 8u), dx, dy from
    _coord_error.  Bilinear backward: each of the at most K outputs that sample a source pixel changes its weight by at most dx + dy,
    and the fp32 sum of K terms rounds by K u per term: |grad - ref| <= K max|g| (dx + dy + (K + 4) u).
    Nearest: exact wherever the fp64 sample position is farther than dx (dy) from a rounding tie; the backward gets small-integer
    gradients (exact sums) and skips the source pixels next to such ambiguous samples."""
    theta = _sweep_thetas(7919 * H + 31 * W + C)
    n = theta.shape[0]
    g = _gen(H * 1000 + W * 10 + C + nearest)
    x = torch.randn(n, C, H, W, generator=g, device=DEV)
    dx, dy = _coord_error(theta, H, W)
    out = _warp(1, x, theta, nearest)
    ref = _ref64(x, theta, nearest)
    ix, iy = _pixel_coords64(theta, H, W)
    K = _window_bound(H, W)
    if not nearest:
        xmax = x.abs().flatten(1).max(1).values.double()
        bar = xmax * (2.0 * (dx + dy) + 8.0 * U)
        err = (out.double() - ref).abs().flatten(1).max(1).values
        assert bool((err <= bar).all()), (err.tolist(), bar.tolist())
        gout = torch.randn(n, C, H, W, generator=g, device=DEV)
        got = _warp(0, gout, theta, nearest)
        want = _ref64_backward(gout, theta, nearest)
        gmax = gout.abs().flatten(1).max(1).values.double()
        bar = K * gmax * (dx + dy + (K + 4) * U)
        err = (got.double() - want).abs().flatten(1).max(1).values
        assert bool((err <= bar).all()), (err.tolist(), bar.tolist())
        return
    near_tie = ((ix - ix.floor() - 0.5).abs() <= dx.view(-1, 1, 1)) | ((iy - iy.floor() - 0.5).abs() <= dy.view(-1, 1, 1))
    clear = ~near_tie                                                    # (n, H, W)
    assert float(clear.float().mean()) > 0.99
    same = (out.double() == ref) | ~clear.unsqueeze(1)
    assert bool(same.all()), int((~same).sum())
    gout = _ints((n, C, H, W), -8, 8, g)
    got = _warp(0, gout, theta, nearest)
    want = _ref64_backward(gout, theta, nearest)
    # source pixels an ambiguous sample may round to: the four around its position
    skip = torch.zeros(n, H, W, dtype=torch.bool, device=DEV)
    m, j, i = near_tie.nonzero(as_tuple=True)
    for ox in (0, 1):
        for oy in (0, 1):
            px = ix[m, j, i].floor().long() + ox
            py = iy[m, j, i].floor().long() + oy
            ok = (px >= 0) & (px < W) & (py >= 0) & (py < H)
            skip[m[ok], py[ok], px[ok]] = True
    same = (got.double() == want) | skip.unsqueeze(1)
    assert bool(same.all()), int((~same).sum())


# ==== B. exact cases ===============================================================================================================
def _dyadic_thetas(H, W):
    """Maps whose every sample position is exact in fp32 on power-of-two maps.  A shift of t in theta moves the sample by t W / 2
    pixels along x (t H / 2 along y)."""
    px, py = 2.0 / W, 2.0 / H                                            # one pixel
    rows = [
        IDENTITY,
        [0.0, -1.0, 0.0, 1.0, 0.0, 0.0],                                 # quarter turns
        [-1.0, 0.0, 0.0, 0.0, -1.0, 0.0],
        [0.0, 1.0, 0.0, -1.0, 0.0, 0.0],
        [1.0, 0.0, 3 * px, 0.0, 1.0, -2 * py],                           # integer shifts
        [-1.0, 0.0, (W - 2) * px, 0.0, -1.0, 0.0],                       # a half turn shifted almost out of the map
        [1.0, 0.0, 0.5 * px, 0.0, 1.0, 0.0],                             # half-pixel shifts: ties of nearest, weights 1/2 and 1/4
        [1.0, 0.0, 0.0, 0.0, 1.0, -0.5 * py],
        [1.0, 0.0, -0.5 * px, 0.0, 1.0, 0.5 * py],
        [1.0, 0.0, 2.5 * px, 0.0, 1.0, 1.5 * py],
        [0.0, -1.0, 0.5 * px, 1.0, 0.0, 0.5 * py],                       # a quarter turn and half-pixel shifts
        [-1.0, 0.0, -1.5 * px, 0.0, -1.0, 2.5 * py],
    ]
    return torch.tensor(rows, dtype=torch.float32, device=DEV).view(-1, 2, 3)


@pytest.mark.parametrize("nearest", [0, 1], ids=["bilinear", "nearest"])
@pytest.mark.parametrize("H,W,C", [(8, 8, 1), (4, 16, 9), (16, 32, 33), (32, 16, 8), (64, 64, 64)])
def test_dyadic_maps_are_bit_exact(H, W, C, nearest):
    """Small integers times weights that are multiples of 1/4: every product and sum is exact, so forward and backward must equal
    fp64 bit for bit, tie rule included."""
    theta = _dyadic_thetas(H, W)
    n = theta.shape[0]
    g = _gen(17 * H + W + C)
    x = _ints((n, C, H, W), -8, 8, g)
    assert torch.equal(_warp(1, x, theta, nearest), _ref64(x, theta, nearest).float())
    gout = _ints((n, C, H, W), -8, 8, g)
    assert torch.equal(_warp(0, gout, theta, nearest), _ref64_backward(gout, theta, nearest).float())


def test_half_pixel_nearest_rounds_half_to_even():
    """The tie rule spelled out: a shift of half a pixel to the right makes output column i sample i + 1/2, which rounds to the even
    neighbour; a shift of half a pixel to the left makes it sample i - 1/2."""
    H, W = 1, 8
    x = torch.arange(W, dtype=torch.float32, device=DEV).view(1, 1, H, W) + 1.0
    for shift, want in ((0.5, [1, 3, 3, 5, 5, 7, 7, 0]), (-0.5, [1, 1, 3, 3, 5, 5, 7, 7])):
        theta = torch.tensor([1.0, 0.0, shift * 2.0 / W, 0.0, 1.0, 0.0], device=DEV).view(1, 2, 3)
        got = _warp(1, x, theta, 1).view(-1).tolist()
        assert got == [float(v) for v in want], (shift, got)


# ==== C. the adjoint as the exact transpose of the forward ======================================================================
@pytest.mark.parametrize("nearest", [0, 1], ids=["bilinear", "nearest"])
@pytest.mark.parametrize("H,W", [(13, 11), (200, 200), (400, 200), (200, 400)])
def test_adjoint_is_the_exact_transpose_of_the_forward(H, W, nearest):
    """Source pixels p_s as channels s: x has channel s one-hot at p_s, so forward channel s is column p_s of the forward's sampling
    matrix, exactly (the other taps add exact zeros).  Then grad_x[s, p_s] of the backward on random g must equal sum_q col_s[q] g_s[q],
    computed in fp64.  The adjoint evaluates each weight with the forward's arithmetic and sums at most K (the window bound) non-zero
    terms in fp32: |error| <= K u sum_q |col_s[q] g_s[q]|.  A candidate missing from a window gives an error of w |g|.  Every source
    pixel is probed under three maps: two rotations with moderate translations and one far out of range."""
    P = H * W
    K = _window_bound(H, W)
    S = 1024
    g = _gen(P + nearest)
    probed = 0
    for chunk, p0 in enumerate(range(0, P, S)):
        p = torch.arange(p0, min(P, p0 + S), device=DEV)
        s = p.numel()
        theta = _rotation_thetas(100003 * H + 7 * W + chunk, 2, 1)
        n = theta.shape[0]
        onehot = torch.zeros(s, P, device=DEV)
        onehot[torch.arange(s, device=DEV), p] = 1.0
        x = onehot.view(1, s, H, W).expand(n, s, H, W)                   # map stride 0: every map probes the same pixels
        cols = _warp(1, x, theta, nearest).view(n, s, P)
        gout = torch.randn(n, s, H, W, generator=g, device=DEV)
        gx = _warp(0, gout, theta, nearest).view(n, s, P)
        got = gx[:, torch.arange(s, device=DEV), p].double()             # (n, s)
        prod = cols.double() * gout.view(n, s, P).double()
        want = prod.sum(-1)
        bar = K * U * prod.abs().sum(-1)
        bad = (got - want).abs() > bar
        assert not bool(bad.any()), (chunk, int(bad.sum()), float((got - want).abs().max()))
        probed += int((cols.abs().sum(-1) > 0).sum())
        del onehot, x, cols, gout, gx, prod
    assert probed >= P // 2                                              # the probes are not vacuous: columns with content


# ==== D. layout and contract ====================================================================================================
@pytest.mark.parametrize("H,W,C", [(13, 11, 9), (200, 200, 33), (400, 200, 65)])
def test_map_strides_and_nan_gaps(H, W, C):
    """Input maps with a stride larger than C*H*W and NaN in the gaps (never read: a NaN times a zero weight would show), outputs with
    a larger stride (gaps and margin untouched, checked in _warp): values bit-identical to the dense call, forward and backward."""
    theta = _sweep_thetas(H + W + C)
    n = theta.shape[0]
    chw = C * H * W
    g = _gen(C)
    x = torch.randn(n, C, H, W, generator=g, device=DEV)
    pad = torch.full((n, chw + 37), float("nan"), device=DEV)
    pad[:, :chw] = x.view(n, chw)
    xs = pad[:, :chw].view(n, C, H, W)
    assert xs.stride(0) == chw + 37
    for nearest in (0, 1):
        for forward in (1, 0):
            dense = _warp(forward, x, theta, nearest)
            assert torch.equal(_warp(forward, xs, theta, nearest, out_stride=chw + 51), dense)
            assert torch.equal(_warp(forward, xs, theta, nearest, out_stride=2 * chw + 3), dense)


@pytest.mark.parametrize("H,W,C", [(13, 11, 33), (200, 200, 64), (400, 200, 65)])
def test_copy_mask_mixed_within_one_call(H, W, C):
    """Maps flagged in the copy mask pass through bit for bit, forward and backward; the others are exactly what a call without a
    mask gives."""
    theta = _sweep_thetas(3 * H + C)
    n = theta.shape[0]
    mask = torch.tensor([1, 0, 1, 0][:n], dtype=torch.uint8, device=DEV)
    g = _gen(H + C)
    x = torch.randn(n, C, H, W, generator=g, device=DEV)
    for nearest in (0, 1):
        for forward in (1, 0):
            got = _warp(forward, x, theta, nearest, mask=mask)
            plain = _warp(forward, x, theta, nearest)
            for m in range(n):
                assert torch.equal(got[m], x[m] if mask[m] else plain[m]), (nearest, forward, m)


def test_zero_maps_change_nothing():
    lib = _lib.load()
    buf = torch.full((64,), float("nan"), device=DEV)
    src = torch.randn(64, device=DEV)
    th = torch.tensor(IDENTITY, device=DEV)
    for fn in (lib.fiery_warp_features_forward, lib.fiery_warp_features_backward):
        _lib.check(fn(0, 4, 4, 4, None, 0, None, None, None, 0, 0, _stream()), "n_maps = 0, NULL pointers")
        _lib.check(fn(0, 4, 4, 4, src.data_ptr(), 64, th.data_ptr(), None, buf.data_ptr(), 64, 1, _stream()), "n_maps = 0")
    assert bool(buf.isnan().all())


def test_most_maps_accepted():
    """n_maps = 65535 (the grid's z limit) runs: 1 x 1 maps, each sampled at its own centre under the identity."""
    n = 65535
    x = torch.randn(n, 1, 1, 1, device=DEV)
    theta = torch.tensor(IDENTITY, device=DEV).repeat(n, 1)
    for forward in (1, 0):
        assert torch.equal(_warp(forward, x, theta, 0), x)


@pytest.mark.parametrize("args", [
    (65536, 1, 1, 1),                   # too many maps
    (1, 1, 8192, 16384),                # H*W = 2^27
    (1, 1, 1, 1 << 27),
    (1, 8 * 65535 + 1, 1, 1),           # more than 65535 blocks of 8 channels
    (-1, 1, 1, 1), (1, 0, 1, 1), (1, 1, 0, 1), (1, 1, 1, 0), (1, 1, -3, 5),
])
def test_bad_shapes_are_rejected(args):
    """These fail before any launch, so a one-element buffer is enough."""
    lib = _lib.load()
    buf = torch.full((8,), float("nan"), device=DEV)
    th = torch.tensor(IDENTITY, device=DEV)
    for fn in (lib.fiery_warp_features_forward, lib.fiery_warp_features_backward):
        rc = fn(*args, buf.data_ptr(), 1, th.data_ptr(), None, buf.data_ptr(), 1, 0, _stream())
        assert rc != 0, args
        assert lib.fiery_last_error()
    torch.cuda.synchronize()
    assert bool(buf.isnan().all())


# ==== E. pose algebra ============================================================================================================
def _theta_call(flow, T, cumulative, n_seq):
    """fiery_warp_theta into a NaN-filled theta and a copy mask filled with 7: every entry must be written."""
    lib = _lib.load()
    n = n_seq * (T if cumulative else 1)
    theta = torch.full((n, 2, 3), float("nan"), device=DEV)
    mask = torch.full((n,), 7, dtype=torch.uint8, device=DEV)
    f = flow.float().contiguous().to(DEV)
    _lib.check(lib.fiery_warp_theta(n_seq, T, cumulative, f.data_ptr(), EXT, 0.5 * EXT, theta.data_ptr(), mask.data_ptr(),
                                    _stream()), "fiery_warp_theta")
    assert not bool(theta.isnan().any()) and not bool((mask == 7).any())
    return theta.cpu(), mask.cpu()


def _pose_flows(n_seq, T, seed, yaw=0.08):
    """Driving-like ego motion with roll and pitch large enough that the order of the Euler product shows."""
    rng = np.random.default_rng(seed)
    f = np.zeros((n_seq, T, 6), np.float32)
    f[..., 0] = rng.uniform(2.5, 7.5, (n_seq, T))
    f[..., 1] = rng.normal(0.0, 0.5, (n_seq, T))
    f[..., 2] = rng.normal(0.0, 0.05, (n_seq, T))
    f[..., 3:5] = rng.normal(0.0, 0.05, (n_seq, T, 2))
    f[..., 5] = rng.normal(0.0, yaw, (n_seq, T))
    return torch.from_numpy(f)


def _theta_bar(flow, T):
    """fp32 against fp64: each entry comes from at most T - 1 products of 4x4 matrices whose rotation entries are at most 1 and whose
    translations add up to at most sum |t| <= S; every product and sincos rounds by a few u relative to those sizes, and theta divides
    the translations by the extent.  Bar: 64 T u (1 + S / extent_y), extent_y the smaller extent."""
    S = float(flow[..., :3].abs().sum(-1).sum(-1).max())
    return 64 * T * U * (1.0 + S / (0.5 * EXT))


@pytest.mark.parametrize("T", [1, 2, 3, 5])
def test_pose_algebra_many_sequences(T):
    """150 sequences (three blocks of 64 threads): cumulative thetas and copy flags against the fp64 oracle."""
    n_seq = 150
    flow = _pose_flows(n_seq, T, seed=T)
    theta, mask = _theta_call(flow, T, 1, n_seq)
    theta, mask = theta.view(n_seq, T, 2, 3), mask.view(n_seq, T)
    assert bool((mask[:, -1] == 1).all()) and bool((mask[:, :-1] == 0).all())
    assert bool((theta[:, -1] == 0).all())
    if T > 1:
        want = WO.cumulative_warp_thetas(flow.double(), (EXT, 0.5 * EXT))
        bar = _theta_bar(flow, T)
        for t in range(T - 1):
            err = float((theta[:, t].double() - want[t]).abs().max())
            assert err <= bar, (t, err, bar)
    plain, pmask = _theta_call(flow[:, 0], 1, 0, n_seq)
    assert bool((pmask == 0).all())
    want = WO.warp_theta(flow[:, 0].double(), (EXT, 0.5 * EXT))
    assert float((plain.double() - want).abs().max()) <= _theta_bar(flow[:, :1], 1)


def test_pose_algebra_yaw_near_pi():
    """Accumulated yaw around +-pi: the atan2 of mat2pose_vec at its branch cut (theta takes cos and sin of it, so either side of
    the cut gives the same map)."""
    n_seq, T = 70, 3
    flow = _pose_flows(n_seq, T, seed=11, yaw=0.01)
    flow[:, :2, 5] += math.pi / 2                                        # frame 0 composes flow[0] and flow[1]: about pi
    flow[::2, :2, 5] *= -1.0                                             # and about -pi; the noise puts it on either side
    theta, _ = _theta_call(flow, T, 1, n_seq)
    theta = theta.view(n_seq, T, 2, 3)
    want = WO.cumulative_warp_thetas(flow.double(), (EXT, 0.5 * EXT))
    bar = _theta_bar(flow, T)
    for t in range(T - 1):
        assert float((theta[:, t].double() - want[t]).abs().max()) <= bar, t
    assert float(want[0][:, 0, 0].min()) < -0.99                         # the composed map did reach a half turn


@pytest.mark.parametrize("F_len", [4, 6])
def test_cumulative_warp_with_a_longer_flow(F_len):
    """A flow longer than the sequence: the reference starts the running product at flow[:, -2] and continues with flow[:, t - 1]
    (the hybrid indexing of warp.py).  Against the CPU oracle, forward and gradient, at the bars of tests/test_warp.py."""
    b, T, C, H, W = 2, 3, 5, 24, 40
    g = torch.Generator().manual_seed(F_len)
    x = torch.randn(b, T, C, H, W, generator=g)
    flow = _pose_flows(b, F_len, seed=F_len, yaw=0.15)
    xd = x.to(DEV).requires_grad_(True)
    out = cumulative_warp_features(xd, flow.to(DEV), mode="bilinear", spatial_extent=(EXT, EXT))
    xo = x.clone().requires_grad_(True)
    ref = WO.cumulative_warp_features(xo.clone(), flow, mode="bilinear", spatial_extent=(EXT, EXT))
    assert float((out.detach().cpu() - ref.detach()).abs().max()) <= 1e-4 * float(ref.detach().abs().max())
    gout = torch.randn(ref.shape, generator=g)
    out.backward(gout.to(DEV))
    ref.backward(gout)
    assert float((xd.grad.cpu() - xo.grad).abs().max()) <= 1e-4 * float(xo.grad.abs().max())


# ==== F. host layer ==============================================================================================================
def _flow_single(n, seed):
    return torch.from_numpy(_flows(np.random.default_rng(seed), n, False)).to(DEV)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("cumulative", [False, True], ids=["warp_features", "cumulative"])
def test_host_half_precision_inputs(dtype, cumulative):
    """fp16 / bf16 x: output and gradient in x's dtype, and equal to the fp32 path on the widened input, rounded."""
    g = _gen(5)
    shape = (2, 3, 9, 20, 24) if cumulative else (3, 9, 20, 24)
    x = torch.randn(*shape, generator=g, device=DEV).to(dtype)
    gout = torch.randn(*shape, generator=g, device=DEV).to(dtype)
    fn = cumulative_warp_features if cumulative else warp_features
    flow = _pose_flows(2, 3, seed=3).to(DEV) if cumulative else _flow_single(3, 5)
    for mode in ("bilinear", "nearest"):
        x16 = x.clone().requires_grad_(True)
        out = fn(x16, flow, mode=mode, spatial_extent=(EXT, EXT))
        out.backward(gout)
        assert out.dtype == dtype and x16.grad.dtype == dtype
        x32 = x.float().requires_grad_(True)
        out32 = fn(x32, flow, mode=mode, spatial_extent=(EXT, EXT))
        out32.backward(gout.float())
        assert torch.equal(out.detach(), out32.detach().to(dtype)), mode
        assert torch.equal(x16.grad, x32.grad.to(dtype)), mode


@pytest.mark.parametrize("cumulative", [False, True], ids=["warp_features", "cumulative"])
def test_host_strided_expanded_and_channels_last_inputs(cumulative):
    """x as a slice of a larger tensor (map stride > C*H*W), expanded along the map dimension (stride 0) and channels-last, and an
    upstream gradient with stride 0: output and gradient bit-identical to the contiguous call."""
    C, H, W = 6, 16, 20
    g = _gen(11)
    fn = cumulative_warp_features if cumulative else warp_features
    lead = (2, 3) if cumulative else (4,)
    flow = _pose_flows(2, 3, seed=9).to(DEV) if cumulative else _flow_single(4, 9)

    def both(x, gout):
        a = x.detach().requires_grad_(True)                             # the layout under test (detach keeps the strides)
        b = x.detach().contiguous().requires_grad_(True)
        outs = []
        for t, gg in ((a, gout), (b, gout.contiguous())):
            out = fn(t, flow, mode="bilinear", spatial_extent=(EXT, EXT))
            out.backward(gg)
            outs.append(out.detach())
        assert torch.equal(outs[0], outs[1])
        assert torch.equal(a.grad, b.grad)
        return outs[0]

    big = torch.randn(*lead, C + 3, H, W, generator=g, device=DEV)
    x = big[..., 1:C + 1, :, :]
    assert x.stride(-3) == H * W and x.stride(-4) == (C + 3) * H * W
    gout = torch.randn(*lead, C, H, W, generator=g, device=DEV)
    both(x, gout)
    one = torch.randn(*([1] * len(lead)), C, H, W, generator=g, device=DEV)
    both(one.expand(*lead, C, H, W), gout)
    if not cumulative:
        both(torch.randn(*lead, C, H, W, generator=g, device=DEV).contiguous(memory_format=torch.channels_last), gout)
    base = torch.randn(*lead, C, H, W, generator=g, device=DEV)
    both(base, torch.tensor(0.75, device=DEV).expand(*lead, C, H, W))
    both(base, torch.randn(C, H, W, generator=g, device=DEV).expand(*lead, C, H, W))

    # the expanded input through autograd: the gradient of the one map is the sum of the per-map gradients
    src = one.clone().requires_grad_(True)
    out = fn(src.expand(*lead, C, H, W), flow, mode="bilinear", spatial_extent=(EXT, EXT))
    out.backward(gout)
    xc = one.expand(*lead, C, H, W).contiguous().requires_grad_(True)
    fn(xc, flow, mode="bilinear", spatial_extent=(EXT, EXT)).backward(gout)
    assert torch.allclose(src.grad, xc.grad.sum(dim=tuple(range(len(lead))), keepdim=True), rtol=1e-6, atol=1e-5)


# ==== G. channel offsets past 2^31 ===============================================================================================
def test_backward_on_a_plane_past_2_pow_31_elements():
    """One 11264 x 11264 map (H*W just under 2^27) with 18 channels: channel c starts c * 126.9 M elements in, past 2^31 from c = 17
    on.  The backward's per-channel offsets must be 64-bit.  With the copy flag set the gradient passes through bit for bit; under the
    identity theta it equals grad_out up to the coordinate error: W (4 + 2) u = 4.0e-3 pixels per axis (_coord_error) moves a weight
    of at most 2 (dx + dy) between neighbours, so |grad_x - grad_out| <= 2 (dx + dy) max|g| + K u max|g|, K = 16.  grad_x starts as NaN
    and must be written everywhere."""
    H = W = 11264
    C = 18
    P = H * W
    assert (C - 1) * P >= 2 ** 31 and P < 2 ** 27
    need = 2 * C * P * 4
    free, _ = torch.cuda.mem_get_info(DEV)
    if free < need + (2 << 30):
        pytest.skip(f"needs about {(need >> 30) + 2} GiB of free device memory, {free >> 30} GiB free")
    lib = _lib.load()
    theta = torch.tensor(IDENTITY, device=DEV)
    gout = torch.empty(C, P, device=DEV)
    gen = _gen(2 ** 27)
    for c in range(C):
        gout[c].normal_(generator=gen)
    gx = torch.empty(C, P, device=DEV)
    dx, dy = _coord_error(theta, H, W)
    bar = float(2.0 * (dx + dy) + 16 * U)
    for copy in (1, 0):
        gx.fill_(float("nan"))
        mask = torch.tensor([copy], dtype=torch.uint8, device=DEV)
        _lib.check(lib.fiery_warp_features_backward(1, C, H, W, gout.data_ptr(), C * P, theta.data_ptr(), mask.data_ptr(),
                                                    gx.data_ptr(), C * P, 0, _stream()), "fiery_warp_features_backward")
        for c in range(C):
            assert not bool(gx[c].isnan().any()), (copy, c)
            if copy:
                assert torch.equal(gx[c], gout[c]), c
            else:
                err = float((gx[c] - gout[c]).abs().max())
                assert err <= bar * float(gout[c].abs().max()), (c, err)
    del gout, gx
    torch.cuda.empty_cache()
