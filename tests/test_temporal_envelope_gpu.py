"""GPU: the temporal tensor-core kernels across the range their C ABI accepts -- the causal convolutions (fiery_b200/csrc/causal_conv.cu)
and the temporal block entry (fiery_b200/csrc/temporal_entry.cu) -- with the cases of tests/_temporal_cases.py.

A  every causal-convolution instantiation (N = 8 .. 64 for the forward, the input gradient and the weight gradient, 1 .. 8 k-steps,
   C_in above and below C_out), bit-exact on small integers against fp64 F.conv3d on the causally padded input;
B  map shapes on, one under and one over the edges of the 8 x 16 output tile and the 32-pixel weight-gradient run;
C  in A, B and D, and for the temporal entry's five blocks: every call goes through the C ABI into guarded buffers -- outputs and
   gradients start as NaN between sentinel margins (every element written, no sentinel touched), the pack and the workspace are
   exactly as large as the *_bytes entry points say, and the inputs lie between NaNs (and, frame-major, with NaN planes in their
   gaps), so a read outside a tensor shows up as a NaN;
D  the weight gradients' chunk rule (csrc/wgrad_chunks.cuh) at 1, 2, 3, 127, 128, 129, 255, 257 and 1009 tiles;
E  operand rounding: with a single 1.0 per channel every output is one product, so it must equal the other operand rounded to TF32
   bit for bit -- to nearest (cvt.rna) for packed weights and for the causal convolution's register operands, and uniformly to
   nearest or uniformly truncated for what the tensor core reads from shared memory as fp32;
F  one shape each whose output offsets pass 2^31 elements;
G  the host layer: channels_last_3d input, an expanded output gradient, bf16 autocast."""
import math

import pytest
import torch
import torch.nn.functional as F

from fiery_b200 import _lib, ops  # noqa: F401
from fiery_b200.causal_conv import conv_backward_data, conv_backward_weight, conv_forward
from fiery_b200.geometry import _stream_ptr
from fiery_b200.temporal import _desc as _entry_desc, _ptrs, _stacked, entry_backward_data, entry_backward_weight, entry_forward
from tests import _temporal_cases as TC
from tests.test_causal_conv_gpu import _reference as _conv_reference
from tests.test_temporal_entry_gpu import BLOCKS, _case as _entry_case, _reference as _entry_reference

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
_ids = lambda v: str(v).replace(" ", "")


@pytest.fixture(autouse=True, scope="module")
def _no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _stream():
    return _stream_ptr(DEV)


def _ints(gen, *shape):
    return torch.randint(-2, 3, shape, generator=gen).float()


# ------------------------------------------------------------------------------------------------------------------------------
# the causal convolution through the C ABI, guarded (C)
# ------------------------------------------------------------------------------------------------------------------------------
def _cc_desc(kt, cin, cout, grid, b, s):
    d = _lib.CausalConv3dDesc()
    d.batch, d.frames, d.grid_x, d.grid_y, d.in_channels, d.out_channels, d.kt = b, s, grid[0], grid[1], cin, cout, kt
    return d


def _cc_pack(d, w):
    """the pack, in a buffer of exactly fiery_causal_conv3d_packed_bytes"""
    lib = _lib.load()
    buf, pack = TC.guarded(int(lib.fiery_causal_conv3d_packed_bytes(d)) // 4, 64, 64, DEV)
    wd = w.to(DEV).contiguous()
    _lib.check(lib.fiery_causal_conv3d_pack_weights(d, wd.data_ptr(), pack.data_ptr(), _stream()), "pack_weights")
    TC.assert_written_and_contained(buf, pack, "pack")
    return pack


def _cc_conv(d, dgrad, inp, w):
    """Forward (x -> y) or input gradient (grad_y -> grad_x) of a poisoned input into a guarded output.  A store that passes the
    row or column guard of the last tile lands at most one 8-row tile past the end: the margin."""
    lib = _lib.load()
    shape = (d.batch, d.in_channels if dgrad else d.out_channels, d.frames, d.grid_x, d.grid_y)
    margin = 8 * d.grid_y + 16
    buf, out = TC.guarded(math.prod(shape), margin, margin, DEV)
    fn = lib.fiery_causal_conv3d_backward_data if dgrad else lib.fiery_causal_conv3d_forward
    src, pack = TC.poisoned(inp, DEV), _cc_pack(d, w)
    _lib.check(fn(d, src.data_ptr(), pack.data_ptr(), out.data_ptr(), _stream()), "conv")
    TC.assert_written_and_contained(buf, out, "input gradient" if dgrad else "output")
    return out.view(shape)


def _cc_wgrad(d, x, gy, fill=float("nan")):
    """The weight gradient of poisoned inputs, its workspace exactly fiery_causal_conv3d_backward_weight_workspace_bytes (holding
    `fill`), followed by one chunk's partial of sentinels."""
    lib = _lib.load()
    n_ws = int(lib.fiery_causal_conv3d_backward_weight_workspace_bytes(d)) // 4
    n_gw = d.out_channels * d.in_channels * d.kt * 9
    wbuf, ws = TC.guarded(n_ws, 64, n_gw + 64, DEV)
    ws.fill_(fill)
    gbuf, gw = TC.guarded(n_gw, 64, 64, DEV)
    xs, gs = TC.poisoned(x, DEV), TC.poisoned(gy, DEV)
    _lib.check(lib.fiery_causal_conv3d_backward_weight(d, xs.data_ptr(), gs.data_ptr(), gw.data_ptr(), ws.data_ptr(), _stream()),
               "backward_weight")
    TC.assert_written_and_contained(wbuf, ws, "workspace", must_write=False)
    TC.assert_written_and_contained(gbuf, gw, "weight gradient")
    return gw.view(d.out_channels, d.in_channels, d.kt, 3, 3)


def _check_causal_exact(kt, ch, grid, b, s):
    cin, cout = ch
    gen = torch.Generator().manual_seed(1000 * kt + 64 * cin + cout + 7 * grid[0] + grid[1] + b + s)
    x, w, gy = _ints(gen, b, cin, s, *grid), _ints(gen, cout, cin, kt, 3, 3), _ints(gen, b, cout, s, *grid)
    y_ref, gx_ref, gw_ref = _conv_reference(x.to(DEV), w.to(DEV), gy.to(DEV))
    d = _cc_desc(kt, cin, cout, grid, b, s)
    assert torch.equal(_cc_conv(d, 0, x, w).double(), y_ref), "forward"
    assert torch.equal(_cc_conv(d, 1, gy, w).double(), gx_ref), "input gradient"
    assert torch.equal(_cc_wgrad(d, x, gy).double(), gw_ref), "weight gradient"


@pytest.mark.parametrize("kt,ch,grid,b,s", TC.A_CASES, ids=_ids)
def test_every_causal_instantiation_bit_exact(kt, ch, grid, b, s):
    _check_causal_exact(kt, ch, grid, b, s)


@pytest.mark.parametrize("kt,ch,grid,b,s", TC.B_CASES, ids=_ids)
def test_causal_map_shapes_against_the_tile_geometry(kt, ch, grid, b, s):
    _check_causal_exact(kt, ch, grid, b, s)


@pytest.mark.parametrize("kt,ch", [(2, (9, 17)), (1, (40, 8))], ids=_ids)
@pytest.mark.parametrize("tiles", TC.D_TILE_COUNTS)
def test_causal_weight_gradient_chunk_edges(tiles, kt, ch):
    b, s, X, Y = TC.D_CAUSAL[tiles]
    _check_causal_exact(kt, ch, (X, Y), b, s)
    gen = torch.Generator().manual_seed(tiles)
    x, gy = torch.randn((b, ch[0], s, X, Y), generator=gen), torch.randn((b, ch[1], s, X, Y), generator=gen)
    d = _cc_desc(kt, *ch, (X, Y), b, s)
    first = _cc_wgrad(d, x, gy)
    for fill in (0.0, 1e30):                                   # the same bits whatever the workspace held
        assert torch.equal(_cc_wgrad(d, x, gy, fill), first), fill


# ------------------------------------------------------------------------------------------------------------------------------
# the temporal entry through the C ABI, guarded (C)
# ------------------------------------------------------------------------------------------------------------------------------
class _Entry:
    """One temporal-entry problem on guarded buffers: x (b, K, s, X, Y) any device, frame-major (strided, NaN planes in the gaps) or
    channel-major; ws the convolutions' (C_q, K + E, 1, 1, 1) weights; extra (b, s, E) or None."""

    def __init__(self, x, ws, extra, layout):
        self.lib = _lib.load()
        self.layout = layout
        self.x = TC.poisoned_frame_major(x, DEV) if layout == "frame_major" else TC.poisoned(x, DEV)
        self.segs = [int(w.shape[0]) for w in ws]
        self.K = int(x.shape[1])
        self.E = int(ws[0].shape[1]) - self.K
        self.extra = TC.poisoned(extra, DEV) if self.E else None
        self.d = _entry_desc(self.x, self.segs, self.E)
        buf, self.pack = TC.guarded(int(self.lib.fiery_temporal_entry_packed_bytes(self.d)) // 4, 64, 64, DEV)
        w = _stacked([t.to(DEV) for t in ws])
        _lib.check(self.lib.fiery_temporal_entry_pack_weights(self.d, w.data_ptr(), self.pack.data_ptr(), _stream()), "pack_weights")
        TC.assert_written_and_contained(buf, self.pack, "pack")

    def _extra_ptr(self):
        return self.extra.data_ptr() if self.E else 0

    def forward(self):
        b, _, s, h, w = self.x.shape
        bufs = [TC.guarded(b * c * s * h * w, 256, 256, DEV) for c in self.segs]
        _lib.check(self.lib.fiery_temporal_entry_forward(self.d, self.x.data_ptr(), self._extra_ptr(), self.pack.data_ptr(),
                                                         _ptrs([v for _, v in bufs]), _stream()), "forward")
        for q, (buf, v) in enumerate(bufs):
            TC.assert_written_and_contained(buf, v, f"output {q}")
        return [v.view(b, c, s, h, w) for (_, v), c in zip(bufs, self.segs)]

    def backward_data(self, grads):
        """grad_x with x's strides; frame-major, the gaps between the frames' channel blocks are sentinels too"""
        buf = torch.full((self.x.numel() * 2 + 2048,), TC.SENTINEL, dtype=torch.float32, device=DEV)
        gx = buf.as_strided(self.x.size(), self.x.stride(), 256)
        gx.fill_(float("nan"))
        gs = [TC.poisoned(g, DEV) for g in grads]
        _lib.check(self.lib.fiery_temporal_entry_backward_data(self.d, _ptrs(gs), self.pack.data_ptr(), gx.data_ptr(), _stream()),
                   "backward_data")
        TC.assert_written_and_contained(buf, gx, "input gradient")
        return gx

    def backward_weight(self, grads, fill=float("nan")):
        n_ws = int(self.lib.fiery_temporal_entry_backward_weight_workspace_bytes(self.d)) // 4
        b, _, s, h, w = self.x.shape
        assert n_ws * 4 == TC.entry_workspace_bytes(b, s, h * w, self.K, self.segs, self.E)
        partial = n_ws // TC.wgrad_chunks(TC.entry_wgrad_tiles(b, s, h * w))
        wbuf, ws = TC.guarded(n_ws, 64, partial + 64, DEV)
        ws.fill_(fill)
        gbuf, gw = TC.guarded(sum(self.segs) * (self.K + self.E), 64, 64, DEV)
        gs = [TC.poisoned(g, DEV) for g in grads]
        _lib.check(self.lib.fiery_temporal_entry_backward_weight(self.d, self.x.data_ptr(), self._extra_ptr(), _ptrs(gs), gw.data_ptr(),
                                                                 ws.data_ptr(), _stream()), "backward_weight")
        TC.assert_written_and_contained(wbuf, ws, "workspace", must_write=False)
        TC.assert_written_and_contained(gbuf, gw, "weight gradient")
        return gw.view(sum(self.segs), self.K + self.E)


def _check_entry_exact(name, grid, b, s, layout, seed):
    x, ws, extra, grads = _entry_case(name, grid, b, s, layout, seed)
    ys_ref, gx_ref, gw_ref = _entry_reference(x, ws, extra, grads)
    e = _Entry(x, ws, extra, layout)
    for q, (y, r) in enumerate(zip(e.forward(), ys_ref)):
        assert torch.equal(y.double(), r), f"output {q}"
    assert torch.equal(e.backward_data(grads).double(), gx_ref), "input gradient"
    assert torch.equal(e.backward_weight(grads).double(), torch.cat([g.flatten(1) for g in gw_ref], 0)), "weight gradient"
    return e, grads


@pytest.mark.parametrize("layout", ["frame_major", "channel_major"])
@pytest.mark.parametrize("grid", [(2, 2), (52, 49), (8, 8)], ids=_ids)
@pytest.mark.parametrize("name", list(BLOCKS))
def test_entry_guarded_and_poisoned(name, grid, layout):
    _check_entry_exact(name, grid, 2, 2, layout, seed=len(name) + grid[0])


@pytest.mark.parametrize("name", ["narrow", "first"])
@pytest.mark.parametrize("tiles", TC.D_TILE_COUNTS)
def test_entry_weight_gradient_chunk_edges(tiles, name):
    b, s, grid = TC.D_ENTRY[tiles]
    _check_entry_exact(name, grid, b, s, "frame_major" if tiles % 2 else "channel_major", seed=tiles)
    x, ws, extra, grads = _entry_case(name, grid, b, s, "channel_major", seed=tiles, ints=False)
    e = _Entry(x, ws, extra, "channel_major")
    first = e.backward_weight(grads)
    for fill in (0.0, 1e30):
        assert torch.equal(e.backward_weight(grads, fill), first), fill


# ------------------------------------------------------------------------------------------------------------------------------
# E: operand rounding
# ------------------------------------------------------------------------------------------------------------------------------
def _which(got, expect, what):
    """got equals expect(tf32_rna) or expect(tf32_trunc) over the whole tensor -- not a mixture; returns and prints which"""
    r, t = expect(TC.tf32_rna), expect(TC.tf32_trunc)
    assert not torch.equal(r, t)
    got = got.cpu()
    is_r, is_t = torch.equal(got, r), torch.equal(got, t)
    assert is_r or is_t, f"{what}: of {got.numel()} elements {int((got != r).sum())} differ from the operand rounded to nearest and " \
                         f"{int((got != t).sum())} from the operand truncated"
    print(f"{what}: the tensor core's shared-memory fp32 operand is {'rounded to nearest' if is_r else 'truncated'} to TF32 "
          f"({torch.cuda.get_device_name(DEV)})")
    return "rna" if is_r else "trunc"


@pytest.mark.parametrize("kt", [1, 2])
@pytest.mark.parametrize("c", [35, 64, 17])
def test_causal_register_operands_are_rounded_to_nearest(c, kt):
    """Permutation weights: y is x, grad_x is grad_y, rounded with cvt.rna on the way out of shared memory and shifted by the tap.
    Every input channel carries a 1.0, so all four fragment registers of every k-step are read."""
    w, where = TC.permutation_weight(c, c, kt, seed=c + kt)
    assert set(where[:, 0].tolist()) == set(range(c))
    b, s, grid = 2, 3, (9, 20)
    x, gy = TC.full_mantissa((b, c, s, *grid), seed=c), TC.full_mantissa((b, c, s, *grid), seed=c + 1)
    d = _cc_desc(kt, c, c, grid, b, s)
    assert torch.equal(_cc_conv(d, 0, x, w).cpu(), TC.shifted_forward(TC.tf32_rna(x), where, kt)), "forward"
    assert torch.equal(_cc_conv(d, 1, gy, w).cpu(), TC.shifted_backward(TC.tf32_rna(gy), where, kt, c)), "input gradient"


@pytest.mark.parametrize("kt", [1, 2])
@pytest.mark.parametrize("ch", [(35, 35), (17, 48), (64, 9)], ids=_ids)
def test_causal_weights_are_rounded_to_nearest_when_packed(ch, kt):
    """An input (output gradient) with a single 1.0 per channel, each in its own 3 x 3 cell: every weight of the forward pack (of the
    transposed pack) comes out once."""
    cin, cout = ch
    w = TC.full_mantissa((cout, cin, kt, 3, 3), seed=cin + cout + kt)
    x = TC.cell_one_hot(cin, kt, 0)
    y = _cc_conv(_cc_desc(kt, cin, cout, tuple(x.shape[-2:]), 1, kt), 0, x, w)
    assert torch.equal(y.cpu(), TC.weights_as_output(TC.tf32_rna(w))), "forward pack"
    gy = TC.cell_one_hot(cout, kt, kt - 1)
    gx = _cc_conv(_cc_desc(kt, cin, cout, tuple(gy.shape[-2:]), 1, kt), 1, gy, w)
    assert torch.equal(gx.cpu(), TC.weights_as_input_gradient(TC.tf32_rna(w))), "transposed pack"


@pytest.mark.parametrize("kt", [1, 2])
@pytest.mark.parametrize("ch", [(35, 35), (17, 48), (64, 9)], ids=_ids)
def test_causal_weight_gradient_operands(ch, kt):
    """grad_y with a single 1.0 per output channel: grad_w is the x each tap reads, rounded with cvt.rna (the register operand).  x
    with a single 1.0 per input channel: grad_w is grad_y as the tensor core reads it from shared memory."""
    cin, cout = ch
    b, s, grid = 2, 3, (9, 40)
    d = _cc_desc(kt, cin, cout, grid, b, s)
    x = TC.full_mantissa((b, cin, s, *grid), seed=cin + kt)
    pos = TC.one_hot_positions(cout, b, s, *grid, seed=cout)
    gw = _cc_wgrad(d, x, TC.one_hot(pos, b, s, *grid))
    assert torch.equal(gw.cpu(), TC.taps_of_x(TC.tf32_rna(x), pos, kt)), "register operand x"
    gy = TC.full_mantissa((b, cout, s, *grid), seed=cout + kt)
    pos = TC.one_hot_positions(cin, b, s, *grid, seed=cin)
    gw = _cc_wgrad(d, TC.one_hot(pos, b, s, *grid), gy)
    _which(gw, lambda rnd: TC.taps_of_grad(rnd(gy), pos, kt), "causal conv weight gradient, grad_y")


def _split(w, segs):
    return [t.reshape(t.shape[0], -1, 1, 1, 1).contiguous() for t in w.split(segs, 0)]


@pytest.mark.parametrize("name", ["first", "limits", "narrow"])
def test_entry_weights_are_rounded_to_nearest_when_packed(name):
    """x (output gradient) with a single 1.0 per channel, channel k at pixel k: y[o, pixel k] = grad_x[k, pixel o] = W[o, k]"""
    K, segs, E = BLOCKS[name]
    n_out, grid = sum(segs), (16, 16)
    w = TC.full_mantissa((n_out, K + E), seed=K)
    want = TC.tf32_rna(w)
    x = torch.zeros(1, K, 1, 256)
    x[0, torch.arange(K), 0, torch.arange(K)] = 1.0
    e = _Entry(x.view(1, K, 1, *grid), _split(w, segs), torch.zeros(1, 1, E) if E else None, "channel_major")
    y = torch.cat([v.flatten(3) for v in e.forward()], 1).cpu()
    assert torch.equal(y[0, :, 0, :K], want[:, :K]) and int(torch.count_nonzero(y[0, :, 0, K:])) == 0
    g = torch.zeros(1, n_out, 1, 256)
    g[0, torch.arange(n_out), 0, torch.arange(n_out)] = 1.0
    gx = e.backward_data([t.reshape(1, -1, 1, *grid) for t in g.split(segs, 1)]).flatten(3).cpu()
    assert torch.equal(gx[0, :, 0, :n_out], want[:, :K].t()) and int(torch.count_nonzero(gx[0, :, 0, n_out:])) == 0


@pytest.mark.parametrize("name", ["first", "limits", "narrow"])
def test_entry_activation_operands(name):
    """Weights with a single 1.0 per output row (at a different input channel each, all of them when N_out >= K): y is x, grad_x is
    grad_y, as the tensor core reads fp32 -- uniformly truncated or uniformly rounded to nearest."""
    K, segs, E = BLOCKS[name]
    n_out, n, b, s, grid = sum(segs), min(sum(segs), K), 2, 2, (8, 12)
    perm = torch.randperm(K, generator=torch.Generator().manual_seed(K))[:n]
    w = torch.zeros(n_out, K + E)
    w[torch.arange(n), perm] = 1.0
    x = TC.full_mantissa((b, K, s, *grid), seed=n_out)
    e = _Entry(x, _split(w, segs), torch.zeros(b, s, E) if E else None, "frame_major")

    def fwd(rnd):
        y = torch.zeros(b, n_out, s, *grid)
        y[:, :n] = rnd(x)[:, perm]
        return y
    _which(torch.cat(e.forward(), 1), fwd, f"temporal entry forward ({name}), x")
    g = TC.full_mantissa((b, n_out, s, *grid), seed=n_out + 1)

    def bwd(rnd):
        gx = torch.zeros(b, K, s, *grid)
        gx[:, perm] = rnd(g)[:, :n]
        return gx
    _which(e.backward_data(list(g.split(segs, 1))), bwd, f"temporal entry input gradient ({name}), grad_y")


@pytest.mark.parametrize("name", ["first", "limits", "narrow"])
def test_entry_weight_gradient_operands_and_egopose(name):
    """grad_y with a single 1.0 per output channel: grad_w's row is the x of that pixel as the tensor core reads it, and its egopose
    columns the frame's egopose rounded with cvt.rna (it is written TF32-rounded into the input tile).  x with a single 1.0 per
    input channel: grad_w's column is grad_y at that pixel.  A single 1.0 in the egopose columns of the weight: the forward's bias is
    fp32 arithmetic, so y is the egopose value unrounded."""
    K, segs, E = BLOCKS[name]
    n_out, b, s, grid = sum(segs), 2, 3, (8, 12)
    x = TC.full_mantissa((b, K, s, *grid), seed=K + 2)
    extra = TC.full_mantissa((b, s, E), seed=K + 3) if E else None
    w0 = torch.zeros(n_out, K + E)
    pos = TC.one_hot_positions(n_out, b, s, *grid, seed=n_out)
    e = _Entry(x, _split(w0, segs), extra, "frame_major")
    gw = e.backward_weight(list(TC.one_hot(pos, b, s, *grid).split(segs, 1)))
    at = lambda t, p: t[p[:, 0], :, p[:, 1], p[:, 2], p[:, 3]]                 # (channels of p, channels of t)
    _which(gw[:, :K], lambda rnd: at(rnd(x), pos), f"temporal entry weight gradient ({name}), x")
    if E:
        assert torch.equal(gw[:, K:].cpu(), TC.tf32_rna(extra)[pos[:, 0], pos[:, 1]]), "egopose columns"
    g = TC.full_mantissa((b, n_out, s, *grid), seed=K + 4)
    pos = TC.one_hot_positions(K, b, s, *grid, seed=K)
    e = _Entry(TC.one_hot(pos, b, s, *grid), _split(w0, segs), torch.zeros(b, s, E) if E else None, "channel_major")
    gw = e.backward_weight(list(g.split(segs, 1)))
    _which(gw[:, :K], lambda rnd: at(rnd(g), pos).t(), f"temporal entry weight gradient ({name}), grad_y")
    if E:
        assert int(torch.count_nonzero(gw[:, K:])) == 0
        w1 = w0.clone()
        w1[torch.arange(n_out), K + torch.arange(n_out) % E] = 1.0
        ys = torch.cat(_Entry(x, _split(w1, segs), extra, "frame_major").forward(), 1).cpu()
        want = extra[:, :, torch.arange(n_out) % E].permute(0, 2, 1)[..., None, None].expand(b, n_out, s, *grid)
        assert torch.equal(ys, want), "egopose bias"


# ------------------------------------------------------------------------------------------------------------------------------
# F: offsets past 2^31 elements
# ------------------------------------------------------------------------------------------------------------------------------
def _need_memory(gib=30):
    free = torch.cuda.mem_get_info(DEV)[0]
    if free < gib * 2 ** 30:
        pytest.skip(f"needs {gib} GiB of free device memory, {free / 2 ** 30:.1f} GiB are free")


def _device_ints(gen, *shape):
    return torch.empty(shape, device=DEV).random_(-2, 3, generator=gen)


def test_causal_offsets_past_2_31_elements():
    """8 -> 64 channels, kt = 2, 3 x 3 frames of 2048 x 2048: 2.4 G output elements.  The reference is fp32 cuDNN with TF32 off, exact
    on small integers, one (batch, frame) slice at a time."""
    _need_memory()
    kt, cin, cout, b, s, X, Y = 2, 8, 64, 3, 3, 2048, 2048
    gen = torch.Generator(device=DEV).manual_seed(0)
    x, w = _device_ints(gen, b, cin, s, X, Y), _device_ints(gen, cout, cin, kt, 3, 3)
    y = conv_forward(x, w)
    assert y.numel() > 2 ** 31

    def padded(xs):                                            # frames t - 1 .. t of one batch element, causally padded
        return F.pad(xs, (1, 1, 1, 1, kt - xs.shape[2], 0))
    for bb in range(b):
        for t in range(s):
            ref = F.conv3d(padded(x[bb:bb + 1, :, max(t - 1, 0):t + 1]), w)
            assert torch.equal(y[bb, :, t], ref[0, :, 0]), (bb, t)
            del ref
    for bb in range(b):                                        # the output-sized tensor becomes grad_y
        y[bb].random_(-2, 3, generator=gen)
    gx = conv_backward_data(y, tuple(x.shape), w)
    gw = conv_backward_weight(y, x, w)
    gx_ref, gw_ref = torch.zeros_like(x), torch.zeros_like(w, dtype=torch.float64)
    for bb in range(b):
        for t in range(s):
            lo = max(t - 1, 0)
            xs, wr = x[bb:bb + 1, :, lo:t + 1].clone().requires_grad_(True), w.clone().requires_grad_(True)
            g_x, g_w = torch.autograd.grad(F.conv3d(padded(xs), wr), (xs, wr), y[bb:bb + 1, :, t:t + 1].contiguous())
            gx_ref[bb, :, lo:t + 1] += g_x[0]
            gw_ref += g_w.double()
            del g_x, g_w, xs
    assert torch.equal(gx, gx_ref), "input gradient"
    assert torch.equal(gw.double(), gw_ref), "weight gradient"
    del x, y, gx, gx_ref
    torch.cuda.empty_cache()


def test_entry_offsets_past_2_31_elements():
    """K = 8 into one 64-channel convolution over the same 3 x 3 x 2048 x 2048 pixels; the reference is an fp32 matrix product per
    frame, exact on small integers."""
    _need_memory()
    K, C, b, s, X, Y = 8, 64, 3, 3, 2048, 2048
    gen = torch.Generator(device=DEV).manual_seed(1)
    x, w = _device_ints(gen, b, K, s, X, Y), _device_ints(gen, C, K, 1, 1, 1)
    w2 = w.view(C, K)
    (y,) = entry_forward(x, [w])
    assert y.numel() > 2 ** 31
    for bb in range(b):
        for t in range(s):
            assert torch.equal(y[bb, :, t].reshape(C, -1), w2 @ x[bb, :, t].reshape(K, -1)), (bb, t)
    for bb in range(b):
        y[bb].random_(-2, 3, generator=gen)
    gx = entry_backward_data([y], x, [w])
    (gw,) = entry_backward_weight([y], x, [w])
    gw_ref = torch.zeros((C, K), dtype=torch.float64, device=DEV)
    for bb in range(b):
        for t in range(s):
            g = y[bb, :, t].reshape(C, -1)
            assert torch.equal(gx[bb, :, t].reshape(K, -1), w2.t() @ g), (bb, t)
            gw_ref += (g @ x[bb, :, t].reshape(K, -1).t()).double()
            del g
    assert torch.equal(gw.view(C, K).double(), gw_ref), "weight gradient"
    del x, y, gx
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------------
# G: host layer
# ------------------------------------------------------------------------------------------------------------------------------
def test_host_layer_layouts_expanded_gradient_and_bf16_autocast():
    gen = torch.Generator().manual_seed(12)
    x, w = _ints(gen, 2, 35, 3, 9, 12).to(DEV), _ints(gen, 32, 35, 2, 3, 3).to(DEV)
    ge = _ints(gen, 1, 32, 1, 1, 12).to(DEV).expand(2, 32, 3, 9, 12)             # stride 0 over batch, frames and rows
    want_y, want_gx, want_gw = _conv_reference(x, w, ge)
    y = conv_forward(x, w)
    assert torch.equal(y.double(), want_y)
    xcl = x.contiguous(memory_format=torch.channels_last_3d)
    assert not xcl.is_contiguous()
    assert torch.equal(conv_forward(xcl, w), y) and torch.equal(torch.ops.fiery_b200.causal_conv3d(xcl, w), y)

    def step(xin, g, autocast=None):
        xi, wi = xin.detach().clone(memory_format=torch.preserve_format).requires_grad_(True), w.detach().clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=autocast or torch.bfloat16, enabled=autocast is not None):
            out = torch.ops.fiery_b200.causal_conv3d(xi, wi)
        assert out.dtype == torch.float32 and torch.equal(out, y)
        out.backward(g)
        return xi.grad, wi.grad
    for xin, g, autocast in ((x, ge, None), (x, ge.contiguous(), None), (xcl, ge, None), (x, ge, torch.bfloat16)):
        assert ge.stride()[0] == 0
        gx, gw = step(xin, g, autocast)
        assert torch.equal(gx.double(), want_gx) and torch.equal(gw.double(), want_gw), (tuple(xin.stride()), tuple(g.stride()), autocast)
    with torch.autocast("cuda", dtype=torch.bfloat16):                          # small integers are exact in bf16
        assert torch.equal(torch.ops.fiery_b200.causal_conv3d(x.bfloat16(), w.bfloat16()), y)
