"""Cases and references shared by tests/test_temporal_cases_cpu.py, tests/test_temporal_envelope_gpu.py and
tests/test_temporal_tail_envelope_gpu.py: the shapes that walk the causal convolution's (csrc/causal_conv.cu), the temporal entry's and
the temporal aggregation's (csrc/temporal_entry.cu) accepted range, the host rules those shapes are chosen by (kernel instantiation,
ring depth, tile and chunk counts, workspace size), the spatial sums' summation order (csrc/spatial_sums.cu), guarded and poisoned
buffers, TF32 rounding on bit patterns, and weights / inputs with a single 1.0 per channel whose expected results are made by indexing
alone.  Importable without a GPU: tensors are created on the device the caller names."""
import math

import numpy as np
import torch

SENTINEL = -1.0e30


def round8(c):
    return (c + 7) // 8 * 8


# ------------------------------------------------------------------------------------------------------------------------------
# TF32 on bit patterns
# ------------------------------------------------------------------------------------------------------------------------------
def tf32_rna(t):
    """fp32 -> TF32, nearest with ties away from zero (cvt.rna.tf32.f32): the 13 low mantissa bits are dropped after adding half"""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def tf32_trunc(t):
    """fp32 -> TF32 by dropping the 13 low mantissa bits (what a tensor core does with an fp32 operand it is handed as TF32)"""
    i = t.float().contiguous().view(torch.int32)
    return (i & ~0x1FFF).view(torch.float32)


def full_mantissa(shape, seed):
    """Random fp32 over 13 binades with all 23 mantissa bits in use, so rounding to nearest and truncation differ on almost every
    element, in both directions; every 7th element is an exact tie (low bits 0x1000), every 11th just below it (0x0FFF), every 13th
    has the low bits all ones."""
    gen = torch.Generator().manual_seed(seed)
    v = torch.randn(shape, generator=gen) * torch.exp2(torch.randint(-6, 7, shape, generator=gen).float())
    i = v.view(torch.int32).flatten()
    for step, low in ((7, 0x1000), (11, 0x0FFF), (13, 0x1FFF)):
        i[::step] = (i[::step] & ~0x1FFF) | low
    return i.view(torch.float32).view(shape)


# ------------------------------------------------------------------------------------------------------------------------------
# causal convolution: case lists.  A case is (kt, (C_in, C_out), (X, Y), batch, frames), as in tests/test_causal_conv_gpu.py
# ------------------------------------------------------------------------------------------------------------------------------
# A: every N = 8 .. 64 as round8(C_in) and as round8(C_out), raw counts on and off the multiple of 8, C_in > C_out and C_in < C_out
A_CHANNELS = [(1, 64), (64, 1), (9, 57), (57, 9), (41, 24), (17, 48), (23, 33), (33, 23), (50, 16), (16, 50), (25, 32), (32, 25),
              (48, 56), (56, 17)]
A_GRIDS = [(7, 12), (52, 48)]
A_CASES = [(kt, ch, grid, (1, 2, 3)[(i + j) % 3], (1, 2, 3)[(i + j + kt) % 3])
           for kt in (1, 2) for i, ch in enumerate(A_CHANNELS) for j, grid in enumerate(A_GRIDS)]

# B: map shapes against the tile geometry (forward / input gradient: 8 x 16 tiles; weight gradient: 32-pixel runs).  Every Y meets
# two X, every X at least two Y, every X % 8 class every Y % 16 class; batch and frames are 2 so a wrong frame or batch coordinate
# reads a neighbour that holds data
B_CHANNELS = [(35, 35), (17, 48)]
B_X = [1, 2, 7, 8, 9, 15, 16, 17]
B_Y = [4, 8, 12, 16, 20, 24, 28, 32, 36, 44, 56, 60, 64, 68]
B_GRIDS = sorted({(B_X[(3 * j + d) % len(B_X)], y) for j, y in enumerate(B_Y) for d in (0, 2)})
B_CASES = [(kt, ch, grid, 2, 2) for kt in (1, 2) for ch in B_CHANNELS for grid in B_GRIDS]


def instantiations(cases):
    """The (kernel, N, k-steps) a case list reaches, by the host code's rules: the forward runs causal_conv_fwd_kernel<round8(C_out)>
    over round8(C_in) / 8 k-steps, the input gradient the same kernel with <round8(C_in)> over round8(C_out) / 8, the weight gradient
    causal_conv_wgrad_kernel<round8(C_out)> (its k-steps are the 32 pixels of a run: None)."""
    got = set()
    for _, (cin, cout), *_ in cases:
        got.add(("forward", round8(cout), round8(cin) // 8))
        got.add(("dgrad", round8(cin), round8(cout) // 8))
        got.add(("wgrad", round8(cout), None))
    return got


ALL_KERNELS = {(kernel, n) for kernel in ("forward", "dgrad", "wgrad") for n in range(8, 65, 8)}


# ------------------------------------------------------------------------------------------------------------------------------
# weight gradients: tiles, chunks (csrc/wgrad_chunks.cuh) and workspace
# ------------------------------------------------------------------------------------------------------------------------------
WG_MAX_CHUNKS = 128
D_TILE_COUNTS = [1, 2, 3, 127, 128, 129, 255, 257, 1009]
# tile count -> (batch, frames, X, Y) of the causal convolution, (batch, frames, (X, Y)) of the temporal entry
D_CAUSAL = {1: (1, 1, 1, 4), 2: (1, 1, 2, 4), 3: (1, 1, 1, 68), 127: (1, 1, 127, 4), 128: (1, 2, 32, 36), 129: (1, 3, 43, 4),
            255: (3, 5, 17, 4), 257: (1, 1, 257, 32), 1009: (1, 1, 1009, 4)}
D_ENTRY = {1: (1, 1, (2, 2)), 2: (1, 1, (8, 16)), 3: (3, 1, (8, 8)), 127: (1, 1, (127, 64)), 128: (2, 1, (64, 64)),
           129: (1, 1, (3, 2732)), 255: (3, 5, (257, 4)), 257: (1, 257, (2, 2)), 1009: (1009, 1, (2, 2))}


def wgrad_chunks(tiles):
    return min(tiles, WG_MAX_CHUNKS)


def chunk_bounds(tiles):
    """[t0, t1) of every chunk"""
    c = wgrad_chunks(tiles)
    return [(i * tiles // c, (i + 1) * tiles // c) for i in range(c)]


def causal_wgrad_tiles(b, s, X, Y):
    """32-pixel runs of one map row"""
    return b * s * X * -(-Y // 32)


def causal_workspace_bytes(b, s, X, Y, cin, cout, kt):
    return wgrad_chunks(causal_wgrad_tiles(b, s, X, Y)) * 9 * kt * cout * cin * 4


def entry_wgrad_tiles(b, s, pixels):
    """64-pixel tiles of one frame (te_bwd_tiles)"""
    return b * s * -(-pixels // 64)


def entry_workspace_bytes(b, s, pixels, K, segs, E):
    r64 = lambda v: (v + 63) // 64 * 64
    return wgrad_chunks(entry_wgrad_tiles(b, s, pixels)) * r64(sum(round8(c) for c in segs)) * r64(K + E) * 4


# ------------------------------------------------------------------------------------------------------------------------------
# temporal aggregation: launch rules and case list.  A case is (N, path channels, R, (X, Y), batch, frames): N output channels, the
# paths' channel counts, R pooled channels
# ------------------------------------------------------------------------------------------------------------------------------
TE_SMEM_MAX = 232448                               # sm_90 opt-in shared memory per block
TE_SMEM_SLACK = 1024 + 256                         # alignment + barriers
TE_STG_BYTES = 32 * 66 * 4                         # one staging tile: 32 channels x 64 pixels at a 66-float pitch
TE_ROW_TABLE_BYTES = 2 * 256 * (8 + 4)             # the forward's per-warpgroup row table


def _round_up(v, m):
    return (v + m - 1) // m * m


def te_stages(fixed_bytes, stage_bytes):
    """ring depth: as many stages as fit next to the fixed shared memory, at most 4"""
    return min((TE_SMEM_MAX - TE_SMEM_SLACK - fixed_bytes) // stage_bytes, 4)


def aggregation_launches(n, paths, r):
    """The kernels one aggregation case launches, by csrc/temporal_entry.cu's host rules with the roles swapped (K = N, the paths as
    the segments, Npad = sum of round8(C_q)):
      forward      ("aggregation", NCHK, stages): temporal_aggregation_kernel<NCHK>, NCHK = ceil(round32(N) / 64); with R = 0 there
                   is no bias and it is ("dgrad", NCHK, stages), the entry's temporal_entry_dgrad_kernel<NCHK>;
      grad_paths   ("forward", NCH, stages): temporal_entry_fwd_kernel<NCH>, NCH = round64(Npad) / 64;
      grad_weight  ("wgrad", nc, threads, stages): temporal_entry_wgrad_kernel<nc>, nc = round64(N) / 64, one warpgroup per 64 rows.
    stages: what te_stages leaves room for next to each kernel's fixed shared memory (the resident weight pack, staging)."""
    kpad, npad = _round_up(n, 32), sum(round8(c) for c in paths)
    npad32, rows = _round_up(npad, 32), _round_up(npad, 64)
    nchk, nch, nc = (kpad + 63) // 64, rows // 64, _round_up(n, 64) // 64
    dgrad = ("aggregation" if r else "dgrad", nchk, te_stages(nchk * 64 * npad32 * 4 + TE_STG_BYTES, 2 * rows * 128))
    fwd = ("forward", nch, te_stages(nch * 64 * kpad * 4 + 2 * TE_STG_BYTES + TE_ROW_TABLE_BYTES, 4 * kpad * 128))
    wgrad = ("wgrad", nc, 2 * rows, te_stages(64, 2 * (rows + 64 * nc) * 128))
    return dgrad, fwd, wgrad


def aggregation_launch_set(cases):
    return {k for n, paths, r, *_ in cases for k in aggregation_launches(n, paths, r)}


# every launch the rules produce over the accepted range: N = 1 .. 128, Npad = 8 .. 256 (any multiple of 8 is one path's round8),
# with and without pooled channels
ALL_AGG_LAUNCHES = aggregation_launch_set([(n, (npad,), r) for n in range(1, 129) for npad in range(8, 257, 8) for r in (0, 1)])

# the maps: X*Y a multiple of 4; one partial tile (4, 60 pixels), exactly one 64- / 128-pixel tile, 4 pixels over, 4 under, and 40000
AGG_GRIDS = {4: (2, 2), 60: (6, 10), 64: (8, 8), 128: (8, 16), 68: (4, 17), 132: (12, 11), 124: (4, 31), 188: (4, 47),
             40000: (200, 200)}
_AGG = [  # (N, paths, R, pixels, batch, frames), with each path set's Npad
    (1, (1,), 1, 4, 1, 1),                         # Npad 8
    (7, (8,), 0, 60, 2, 3),                        # 8
    (8, (1, 8, 8), 23, 64, 3, 2),                  # 24
    (9, (35, 35, 35), 0, 68, 2, 2),                # 120
    (31, (65, 63), 1, 132, 2, 1),                  # 136
    (32, (48, 48, 48), 0, 124, 1, 2),              # 144
    (33, (57, 64, 3, 100), 23, 188, 1, 2),         # 240
    (63, (100, 100), 0, 128, 1, 3),                # 208 (Npad32 224)
    (64, (33, 31), 200, 40000, 1, 2),              # 72
    (64, (1, 2, 3, 4), 23, 60, 2, 2),              # 32
    (65, (8,), 23, 68, 2, 3),                      # 8
    (96, (35, 35, 35), 0, 132, 2, 2),              # 120
    (80, (65, 63), 23, 124, 1, 3),                 # 136
    (96, (96, 96), 0, 64, 3, 1),                   # 192
    (65, (64, 64, 64, 64), 1, 188, 1, 2),          # 256
    (96, (256,), 0, 40000, 1, 1),                  # 256
    (127, (1, 8, 8), 0, 4, 3, 2),                  # 24
    (128, (33, 31), 23, 128, 2, 2),                # 72
    (127, (48, 48, 48), 200, 40000, 1, 1),         # 144
    (128, (100, 100), 1, 60, 2, 2),                # 208 (Npad32 224): one stage
    (112, (57, 64, 3, 100), 0, 68, 1, 3),          # 240
]
AGG_CASES = [(n, paths, r, AGG_GRIDS[p], b, s) for n, paths, r, p, b, s in _AGG]


# ------------------------------------------------------------------------------------------------------------------------------
# spatial sums: the kernel's summation order
# ------------------------------------------------------------------------------------------------------------------------------
SS_THREADS = 256


def spatial_sums_model(planes, pixels):
    """spatial_sums_kernel's sum of each plane, in its order, in fp32: planes (..., pixels) -> (...) np.float32.  The plane is cut into
    4-pixel chunks (the last one zero-filled); thread i adds chunks i, i + 256, i + 512, ... lane by lane into four accumulators,
    ascending; its total is (a0 + a1) + (a2 + a3); each warp's 32 totals are added by an xor butterfly (offsets 16, 8, 4, 2, 1), and the
    eight warp sums in ascending order.  Threads past the last chunk add nothing: their zero pads here leave every sum as it is."""
    x = np.asarray(planes, dtype=np.float32)
    lead = x.shape[:-1]
    x = x.reshape(-1, pixels)
    rounds = -(-pixels // (4 * SS_THREADS))
    chunks = np.zeros((x.shape[0], rounds * SS_THREADS * 4), np.float32)
    chunks[:, :pixels] = x
    chunks = chunks.reshape(-1, rounds, SS_THREADS, 4)
    acc = np.zeros((x.shape[0], SS_THREADS, 4), np.float32)
    for k in range(rounds):
        acc = acc + chunks[:, k]
    v = ((acc[..., 0] + acc[..., 1]) + (acc[..., 2] + acc[..., 3])).reshape(-1, SS_THREADS // 32, 32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lane ^ o]
    total = v[:, 0, 0]
    for w in range(1, SS_THREADS // 32):
        total = total + v[:, w, 0]
    return total.reshape(lead)


# ------------------------------------------------------------------------------------------------------------------------------
# guarded outputs and poisoned inputs
# ------------------------------------------------------------------------------------------------------------------------------
def _round4(n):
    return (n + 3) // 4 * 4


def guarded(n, front, back, device):
    """(buffer, view): a 16-byte-aligned view of n NaN floats inside a buffer that holds at least `front` sentinels before it and
    `back` after it."""
    front = _round4(front)
    buf = torch.full((front + n + back,), SENTINEL, dtype=torch.float32, device=device)
    view = buf[front:front + n]
    view.fill_(float("nan"))
    assert view.data_ptr() % 16 == 0
    return buf, view


def assert_written_and_contained(buf, view, what, must_write=True):
    """Every element of `view` (any strides, inside the 1-D `buf`) was written, with something other than NaN, and no other element
    of `buf` changed.  must_write=False: only the second half (a workspace may be larger than what the kernel uses)."""
    n_nan = int(view.isnan().sum()) if must_write else 0
    assert n_nan == 0, f"{what}: {n_nan} of {view.numel()} elements were never written or are NaN (a read outside an input)"
    rest = buf.clone()
    rest.as_strided(view.size(), view.stride(), view.storage_offset() - buf.storage_offset()).fill_(SENTINEL)
    bad = (rest != SENTINEL).nonzero().flatten()        # NaN != SENTINEL too
    assert bad.numel() == 0, f"{what}: {bad.numel()} stores outside the tensor, the first at buffer element {int(bad[0])} " \
                             f"(the tensor starts at {view.storage_offset() - buf.storage_offset()})"


def poisoned(t, device, margin=1024):
    """A contiguous fp32 copy of t on `device` with `margin` NaNs before and after it in the same allocation (16-byte aligned): a
    read outside the tensor's own extent turns an output into NaN."""
    margin = _round4(margin)
    buf = torch.full((2 * margin + t.numel(),), float("nan"), dtype=torch.float32, device=device)
    view = buf[margin:margin + t.numel()].view(t.shape)
    view.copy_(t)
    assert view.data_ptr() % 16 == 0
    return view


def poisoned_frame_major(x, device, gap=4, margin=1024):
    """x (b, K, s, X, Y) stored frame-major -- the permuted view TemporalModel.forward makes -- with `gap` NaN channel planes after each
    frame's K and NaN margins around the whole: a strided (b, K, s, X, Y) view."""
    b, k, s, h, w = x.shape
    margin = _round4(margin)
    n = b * s * (k + gap) * h * w
    buf = torch.full((2 * margin + n,), float("nan"), dtype=torch.float32, device=device)
    view = buf[margin:margin + n].view(b, s, k + gap, h, w)[:, :, :k].permute(0, 2, 1, 3, 4)
    view.copy_(x)
    assert view.data_ptr() % 16 == 0
    return view


# ------------------------------------------------------------------------------------------------------------------------------
# causal convolution: a single 1.0 per channel, expectations by indexing
# ------------------------------------------------------------------------------------------------------------------------------
def permutation_weight(c_out, c_in, kt, seed):
    """(weight (c_out, c_in, kt, 3, 3), where (c_out, 4)): exactly one 1.0 per output channel o, at where[o] = (input channel, tau,
    dy, dx), seeded; the input channels cover 0 .. c_in - 1 when c_out >= c_in and the taps all 9 kt when c_out >= 9 kt."""
    gen = torch.Generator().manual_seed(seed)
    taps = 9 * kt
    draw = lambda n: torch.cat([torch.randperm(n, generator=gen) for _ in range(-(-c_out // n))])[:c_out]
    ci, tap = draw(c_in), draw(taps)
    where = torch.stack([ci, tap // 9, tap // 3 % 3, tap % 3], 1)
    w = torch.zeros(c_out, c_in, kt, 3, 3)
    w[torch.arange(c_out), ci, where[:, 1], where[:, 2], where[:, 3]] = 1.0
    assert int(w.sum()) == c_out and bool((w.flatten(1).sum(1) == 1).all())
    assert c_out < c_in or set(ci.tolist()) == set(range(c_in))
    assert c_out < taps or set(tap.tolist()) == set(range(taps))
    return w, where


def _pad_front(x, kt):
    """the forward's zero padding: kt - 1 frames in front, one pixel around the map"""
    b, c, s, h, w = x.shape
    xp = x.new_zeros(b, c, s + kt - 1, h + 2, w + 2)
    xp[:, :, kt - 1:, 1:-1, 1:-1] = x
    return xp


def _pad_back(gy, kt):
    """the input gradient's: kt - 1 frames behind, one pixel around the map"""
    b, c, s, h, w = gy.shape
    gp = gy.new_zeros(b, c, s + kt - 1, h + 2, w + 2)
    gp[:, :, :s, 1:-1, 1:-1] = gy
    return gp


def shifted_forward(x, where, kt):
    """The causal convolution of x with permutation_weight's weight: output channel o is input channel i shifted by its tap, zeros
    where the tap reads the padding."""
    b, _, s, h, w = x.shape
    xp = _pad_front(x, kt)
    return torch.stack([xp[:, i, tau:tau + s, dy:dy + h, dx:dx + w] for i, tau, dy, dx in where.tolist()], 1)


def shifted_backward(gy, where, kt, c_in):
    """The input gradient for permutation_weight's weight when no input channel is used twice: input channel i is output channel
    o's gradient shifted the other way; unused input channels get zeros."""
    b, _, s, h, w = gy.shape
    assert len(set(where[:, 0].tolist())) == where.shape[0], "an input channel used twice would need a sum"
    gp = _pad_back(gy, kt)
    gx = gy.new_zeros(b, c_in, s, h, w)
    for o, (i, tau, dy, dx) in enumerate(where.tolist()):
        gx[:, i] = gp[:, o, kt - 1 - tau:kt - 1 - tau + s, 2 - dy:2 - dy + h, 2 - dx:2 - dx + w]
    return gx


def one_hot_positions(channels, b, s, X, Y, seed):
    """(channels, 4) seeded (batch, frame, x, y), one per channel; the first four sit in the map's corners"""
    gen = torch.Generator().manual_seed(seed)
    pos = torch.stack([torch.randint(0, n, (channels,), generator=gen) for n in (b, s, X, Y)], 1)
    for j, (px, py) in enumerate([(0, 0), (0, Y - 1), (X - 1, 0), (X - 1, Y - 1)][:channels]):
        pos[j, 2], pos[j, 3] = px, py
    return pos


def one_hot(pos, b, s, X, Y):
    """(b, channels, s, X, Y) with 1.0 at pos[c] in channel c, zeros elsewhere"""
    c = pos.shape[0]
    t = torch.zeros(b, c, s, X, Y)
    t[pos[:, 0], torch.arange(c), pos[:, 1], pos[:, 2], pos[:, 3]] = 1.0
    return t


def taps_of_x(x, pos, kt):
    """The weight gradient when grad_y is one_hot(pos) (one 1.0 per output channel): grad_w[o, i, tau, dy, dx] is the input element
    that tap reads for output position pos[o]."""
    xp = _pad_front(x, kt)
    out = []
    for bb, t, px, py in pos.tolist():
        out.append(xp[bb, :, t:t + kt, px:px + 3, py:py + 3])
    return torch.stack(out, 0)


def taps_of_grad(gy, pos, kt):
    """The weight gradient when x is one_hot(pos) (one 1.0 per input channel): grad_w[o, i, tau, dy, dx] is the output gradient at
    the position whose tap reads pos[i]."""
    gp = _pad_back(gy, kt)
    out = []
    for bb, t, px, py in pos.tolist():
        win = gp[bb, :, t:t + kt, px:px + 3, py:py + 3]         # [o, kt - 1 - tau, 2 - dy, 2 - dx]
        out.append(win.flip(1, 2, 3))
    return torch.stack(out, 1)


def cell_grid(channels):
    """(X, Y, pos (channels, 2)): channel c's pixel is the centre of its own 3 x 3 cell of an X x Y map (Y a multiple of 4), so the
    3 x 3 neighbourhoods of different channels do not meet."""
    m = math.isqrt(channels - 1) + 1
    c = torch.arange(channels)
    return 3 * m, (3 * m + 3) // 4 * 4, torch.stack([3 * (c // m) + 1, 3 * (c % m) + 1], 1)


def cell_one_hot(channels, kt, frame):
    """(1, channels, kt, X, Y) with 1.0 at channel c's cell centre in `frame`"""
    X, Y, pos = cell_grid(channels)
    t = torch.zeros(1, channels, kt, X, Y)
    t[0, torch.arange(channels), frame, pos[:, 0], pos[:, 1]] = 1.0
    return t


def weights_as_output(w):
    """The causal convolution of cell_one_hot(C_in, kt, 0) with w: every weight once, w[o, i, tau, dy, dx] at frame kt - 1 - tau,
    pixel cell(i) - (dy - 1, dx - 1) of output channel o."""
    c_out, c_in, kt = w.shape[:3]
    X, Y, pos = cell_grid(c_in)
    y = w.new_zeros(1, c_out, kt, X, Y)
    for i, (px, py) in enumerate(pos.tolist()):
        y[0, :, :, px - 1:px + 2, py - 1:py + 2] = w[:, i].flip(1, 2, 3)
    return y


def weights_as_input_gradient(w):
    """The input gradient for grad_y = cell_one_hot(C_out, kt, kt - 1): w[o, i, tau, dy, dx] at frame tau, pixel cell(o) + (dy - 1,
    dx - 1) of input channel i."""
    c_out, c_in, kt = w.shape[:3]
    X, Y, pos = cell_grid(c_out)
    gx = w.new_zeros(1, c_in, kt, X, Y)
    for o, (px, py) in enumerate(pos.tolist()):
        gx[0, :, :, px - 1:px + 2, py - 1:py + 2] = w[o]
    return gx
