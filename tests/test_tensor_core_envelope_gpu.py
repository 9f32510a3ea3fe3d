"""GPU: the two wgmma kernels (the depth layer, fiery_b200/csrc/depth_layer.cu, and the first BEV convolution,
fiery_b200/csrc/bev_conv.cu) across the shapes their C ABI accepts, the depth layer's autograd backward, and the gradient of the
whole training step, against fp64.

  A. depth layer forward: 1 <= n_out <= 128 (both epilogue guards: the 16-bit path's rows r0 / r0 + 8 and warpgroup 1's channels
     64..127, the fp32 path's channel pairs 8j + cq), fp32 / fp16 / bf16, pixels % 4 == 0 with a 16-byte row pitch, from the
     smallest accepted pixel count to ragged multi-tile images; every persistent-ring wrap; the contract's edges.
  B. depth layer backward (one aten::convolution_backward on the packed, rounded weights) through the module: channels-last
     features, features without grad, a frozen weight, with and without bias.
  C. first BEV convolution: grids where the 7x7 window meets both borders of an axis, a single tile, exact tile multiples, the
     lift's odd grids, every Ho % 8 / Wo % 16 tail class; all four epilogues; conversion paths and edges.
  D. the training step's flat gradient (LiftTrainer, precision 32) against an fp64 replica of the model.

Kernel outputs that are checked value for value go through the C ABI into a NaN-filled buffer followed by a sentinel margin as large
as anything the kernel can address: every output must be written and nothing past the output may change.  References are fp64
convolutions on the GPU; torch's own TF32 is switched off for the whole module, so a torch "reference" is not itself TF32."""
import math

import pytest
import torch
import torch.nn.functional as F

from fiery_b200 import _lib
from fiery_b200.bev_conv import first_conv_forward
from fiery_b200.bev_conv import pack_weight as pack_conv_weight
from fiery_b200.depth_layer import _DTYPE_CODE, DepthLayer, depth_layer_forward
from fiery_b200.depth_layer import pack_weight as pack_depth_weight
from fiery_b200.synthetic import CONFIGS, LiftConfig
from fiery_b200.train import LiftTrainer, synthetic_batch
from oracle import lift_oracle as O

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_ID = {torch.float32: "fp32", torch.float16: "fp16", torch.bfloat16: "bf16"}
SENTINEL = -1.0e30                  # a value no kernel output here can take


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    """torch's convolutions and matmuls in true fp32 (a TF32 'reference' is only good to ~1e-3); the old settings come back after."""
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g, device=DEV).float()


def _nerr(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _tf32(t):
    """fp32 -> the nearest TF32 number (10 explicit mantissa bits, ties away from zero), still stored as fp32."""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & -0x2000).view(torch.float32)


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _guarded(n, margin):
    """A buffer of n NaNs followed by `margin` sentinels."""
    buf = torch.full((n + margin,), float("nan"), device=DEV)
    buf[n:] = SENTINEL
    return buf


def _assert_written_and_contained(buf, n, what):
    assert not bool(buf[:n].isnan().any()), (what, int(buf[:n].isnan().sum()), "outputs never written")
    assert bool((buf[n:] == SENTINEL).all()), (what, "store past the end of the output")


# ==== A. depth layer forward =====================================================================================================
def _dl_call(feat, wp, bias, n_out):
    """fiery_depth_layer_forward on a guarded output.  The kernel addresses rows r < 128 of an image's head and pixels < p0 + 128 of
    its last tile, so no store, guarded or not, can reach past 128 * pixels + 128 floats after the end: that is the margin."""
    N, _, h, w = feat.shape
    P = h * w
    n = N * n_out * P
    buf = _guarded(n, 128 * P + 128)
    _lib.check(_lib.load().fiery_depth_layer_forward(N, P, n_out, feat.data_ptr(), _DTYPE_CODE[feat.dtype], wp.data_ptr(),
                                                     bias.data_ptr() if bias is not None else None, buf.data_ptr(), _stream()),
               "fiery_depth_layer_forward")
    _assert_written_and_contained(buf, n, (DT_ID[feat.dtype], N, P, n_out))
    return buf[:n].view(N, n_out, h, w)


DL_N_OUT = [1, 7, 8, 9, 63, 64, 65, 71, 72, 105, 112, 120, 127, 128]
DL_N_OUT_ALL_PIXELS = (1, 65, 128)
# (h, w) of the pixel counts: the smallest accepted (4 in fp32, 8 in 16 bits), under one tile (12, 120), one tile (128 = 8 x 16, also
# a lift head shape), one tile plus a ragged second (136), the lift envelope's head shapes a dtype accepts (5 x 12, 1 x 60, 3 x 4 and
# 31 x 36 are fp32 only: h*w = 4 mod 8), and the bench's 28 x 60
DL_HW = {
    torch.float32: [(1, 4), (3, 4), (1, 120), (8, 16), (8, 17), (5, 12), (32, 20), (1, 60), (2, 36), (31, 36), (28, 60)],
    torch.float16: [(1, 8), (1, 120), (8, 16), (8, 17), (32, 20), (2, 36), (28, 60)],
}
DL_HW[torch.bfloat16] = DL_HW[torch.float16]
# the pixel subset for the other output counts: the minimum, one tile, one tile + a ragged one, a long ragged image
DL_HW_SUBSET = {torch.float32: [(1, 4), (8, 16), (8, 17), (31, 36)], torch.float16: [(1, 8), (8, 16), (8, 17), (28, 60)]}
DL_HW_SUBSET[torch.bfloat16] = DL_HW_SUBSET[torch.float16]
# normwise bar against the fp64 convolution of the unrounded fp32 operands: the operand type's rounding of features and weights
DL_UNROUNDED_TOL = {torch.float16: 2e-3, torch.bfloat16: 1e-2, torch.float32: 1e-3}


def _dl_operands(dtype, N, h, w, n_out, g):
    """Random operands: fp32 originals, and the operands rounded to what the tensor core multiplies.  In fp32 the kernel multiplies
    TF32, so both are rounded to TF32 first and the 'same rounded operands' reference is exact for it as well."""
    feat = torch.randn(N, 128, h, w, generator=g, device=DEV)
    weight = torch.randn(n_out, 128, 1, 1, generator=g, device=DEV) * 0.1
    bias = torch.randn(n_out, generator=g, device=DEV)
    if dtype == torch.float32:
        feat_r, weight_r = _tf32(feat), _tf32(weight)
    else:
        feat_r, weight_r = feat.to(dtype), weight.to(dtype).float()
    return feat, weight, bias, feat_r, weight_r


@pytest.mark.parametrize("n_out", DL_N_OUT)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_depth_layer_sweep_matches_fp64(dtype, n_out):
    """Against the fp64 convolution of the same rounded operands (products exact, only the fp32 accumulation differs): 1e-5 normwise
    and |got - same| <= 1e-5 * max(sum |w||x| + |b|) element-wise; against the unrounded fp32 operands: the operand type's bar,
    normwise over all shapes of the case."""
    hws = DL_HW[dtype] if n_out in DL_N_OUT_ALL_PIXELS else DL_HW_SUBSET[dtype]
    g = _gen(1000 * n_out + DTYPES.index(dtype))
    err2 = ref2 = 0.0
    for h, w in hws:
        N = 2
        feat, weight, bias, feat_r, weight_r = _dl_operands(dtype, N, h, w, n_out, g)
        wp = pack_depth_weight(weight_r if dtype == torch.float32 else weight, dtype)      # 16 bits: the packing rounds
        for b in (bias, None):
            got = _dl_call(feat_r, wp, b, n_out)
            b64 = b.double() if b is not None else None
            same = F.conv2d(feat_r.double(), weight_r.double(), b64)
            assert _nerr(got, same) < 1e-5, (h, w, b is None, _nerr(got, same))
            scale = F.conv2d(feat_r.double().abs(), weight_r.double().abs())
            if b is not None:
                scale = scale + b.double().abs().view(1, -1, 1, 1)
            worst = float((got.double() - same).abs().max())
            assert worst <= 1e-5 * float(scale.max()), (h, w, b is None, worst, float(scale.max()))
            exact = F.conv2d(feat.double(), weight.double(), b64)
            err2 += float((got.double() - exact).square().sum())
            ref2 += float(exact.square().sum())
    assert math.sqrt(err2 / ref2) < DL_UNROUNDED_TOL[dtype], math.sqrt(err2 / ref2)


# ragged shapes for the integer checks: the smallest pixel count, under one tile, one tile + 8 pixels, multi-tile with a short tail
DL_RAGGED = {torch.float32: [(1, 4), (3, 4), (1, 120), (8, 17), (31, 36), (28, 60)],
             torch.float16: [(1, 8), (1, 120), (8, 17), (2, 36), (28, 60)]}
DL_RAGGED[torch.bfloat16] = DL_RAGGED[torch.float16]


def _dl_int_operands(dtype, N, h, w, n_out, g):
    """Small integers: exact in every operand type, and every partial sum is exact in fp32."""
    feat = _ints((N, 128, h, w), -4, 4, g).to(dtype)
    weight = _ints((n_out, 128, 1, 1), -3, 3, g)
    bias = _ints((n_out,), -8, 8, g)
    return feat, weight, bias


@pytest.mark.parametrize("n_out", [1, 9, 65, 72, 127, 128])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_depth_layer_integers_are_bit_exact(dtype, n_out):
    """Every output equal to the fp32 convolution: catches the swizzle, dl_feat_offset / dl_pixel and channel addressing on a partial
    last tile, in each operand type."""
    g = _gen(31 * n_out + DTYPES.index(dtype))
    for h, w in DL_RAGGED[dtype]:
        feat, weight, bias = _dl_int_operands(dtype, 3, h, w, n_out, g)
        wp = pack_depth_weight(weight, dtype)
        for b in (bias, None):
            want = F.conv2d(feat.double(), weight.double(), b.double() if b is not None else None).float()
            assert torch.equal(_dl_call(feat, wp, b, n_out), want), (h, w, b is None)


@pytest.mark.parametrize("n_out", [1, 65, 127])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_depth_layer_writes_every_output_and_nothing_past_it(dtype, n_out):
    """A ragged image (136 pixels: a full tile and 8 pixels) behind a NaN-filled output and a sentinel margin: no NaN may survive, the
    margin must be intact (checked in _dl_call), and the values must be exact."""
    g = _gen(5 + n_out)
    feat, weight, bias = _dl_int_operands(dtype, 3, 8, 17, n_out, g)
    got = _dl_call(feat, pack_depth_weight(weight, dtype), bias, n_out)
    assert torch.equal(got, F.conv2d(feat.double(), weight.double(), bias.double()).float())


def _dl_stages(dtype):
    return 2 if dtype == torch.float32 else 4         # DlShape<ES>::STAGES: feature tiles in flight


def _dl_schedule(n_tiles, n_sm):
    """Mirror of launch_depth_layer's grid rule (fiery_b200/csrc/depth_layer.cu); the library does not report it, so a change there
    must be made here too.  One persistent CTA per SM: waves = ceil(tiles / SMs), grid = ceil(tiles / waves), and CTA b runs tiles
    b, b + grid, ...  Returns (grid, the most tiles one CTA runs)."""
    waves = -(-n_tiles // n_sm)
    grid = -(-n_tiles // waves)
    return grid, -(-n_tiles // grid)


DL_RING_PICKS = [(dt, k) for dt in DTYPES for k in ("1", "S", "S+1", "2S+1")]


@pytest.mark.parametrize("dtype,ring", DL_RING_PICKS, ids=[f"{DT_ID[d]}-{k}" for d, k in DL_RING_PICKS])
def test_depth_layer_persistent_ring_wraps(dtype, ring):
    """Image counts at which the busiest CTA runs 1, STAGES, STAGES + 1 and 2 * STAGES + 1 tiles: the ring's stage index and its
    full / empty parities wrap once, at the first reuse and at the second.  248 pixels: two tiles per image, the second ragged."""
    S = _dl_stages(dtype)
    want = {"1": 1, "S": S, "S+1": S + 1, "2S+1": 2 * S + 1}[ring]
    n_sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    images = next(n for n in range(1, 4 * want * n_sm) if _dl_schedule(2 * n, n_sm)[1] == want)
    grid, most = _dl_schedule(2 * images, n_sm)
    assert most == want and grid <= n_sm
    g = _gen(want)
    feat, weight, bias = _dl_int_operands(dtype, images, 8, 31, 112, g)
    got = _dl_call(feat, pack_depth_weight(weight, dtype), bias, 112)
    assert torch.equal(got, F.conv2d(feat.double(), weight.double(), bias.double()).float()), (images, grid, most)


def test_depth_layer_contract_edges():
    from fiery_b200._lib import FieryError
    lib = _lib.load()
    feat = torch.zeros(1, 128, 8, 16, device=DEV)
    wp = torch.zeros(128, 128, device=DEV)
    out = torch.full((2 * 129 * 128,), SENTINEL, device=DEV)
    for n_out in (0, 129):
        with pytest.raises(FieryError, match="bad shape"):
            _lib.check(lib.fiery_depth_layer_forward(1, 128, n_out, feat.data_ptr(), 0, wp.data_ptr(), None, out.data_ptr(), _stream()),
                       "fiery_depth_layer_forward")
    # no images: returns before it touches the output
    _lib.check(lib.fiery_depth_layer_forward(0, 128, 64, feat.data_ptr(), 0, wp.data_ptr(), None, out.data_ptr(), _stream()), "n = 0")
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all())
    assert tuple(depth_layer_forward(feat[:0], torch.zeros(64, 128, 1, 1, device=DEV), None).shape) == (0, 64, 8, 16)
    # the 16-bit row pitch: h*w = 4 (mod 8) is rejected in fp16 / bf16 and accepted in fp32 -- the lift's 5 x 12, 3 x 4 and 31 x 36
    # heads under AMP; h*w = 0 (mod 8) is accepted in every type; fp32 needs h*w % 4 == 0
    g = _gen(11)
    for h, w in ((5, 12), (3, 4), (31, 36), (1, 4)):
        assert (h * w) % 8 == 4
        feat, weight, bias = _dl_int_operands(torch.float32, 2, h, w, 70, g)
        want = F.conv2d(feat.double(), weight.double(), bias.double()).float()
        assert torch.equal(depth_layer_forward(feat, weight, bias), want)
        for dtype in (torch.float16, torch.bfloat16):
            with pytest.raises(FieryError, match="16-byte row pitch"):
                depth_layer_forward(feat.to(dtype), weight, bias)
            feat8 = torch.cat([feat, feat[..., :4]], dim=-1)       # four more columns: h*w = 0 (mod 8)
            assert (h * feat8.shape[-1]) % 8 == 0
            ok = depth_layer_forward(feat8.to(dtype), weight, bias)
            assert torch.equal(ok, F.conv2d(feat8.double(), weight.double(), bias.double()).float())
    for h, w in ((1, 2), (1, 6), (3, 2)):
        with pytest.raises(FieryError, match="16-byte row pitch"):
            depth_layer_forward(torch.zeros(1, 128, h, w, device=DEV), torch.zeros(8, 128, 1, 1, device=DEV), None)


# ==== B. depth layer backward ====================================================================================================
# unit roundoff of the type the backward computes in: the upstream gradient is rounded to it, and so are g_feat and g_weight
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}


def _assert_grad_bound(got, want, absterms, u, k, what):
    """Element-wise bound for a k-term sum of products computed with the upstream gradient rounded to the operand type (<= u
    relative per term), fp32 accumulation (<= k * 2^-24 of the sum of |terms|) and the result rounded to the operand type (<= u):
    |got - want| <= (2u + k * 2^-24) * sum |terms|."""
    assert got is not None and got.shape == want.shape, what
    bar = (2 * u + k * 2.0 ** -24) * absterms
    excess = (got.double() - want).abs() - bar
    assert float(excess.max()) <= 0, (what, float(((got.double() - want).abs() / bar.clamp_min(1e-300)).max()))
    assert float(want.abs().max()) > 0, what


@pytest.mark.parametrize("route", ["contiguous", "channels_last", "feature_input", "frozen_weight"])
@pytest.mark.parametrize("has_bias", [True, False], ids=["bias", "no_bias"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_depth_layer_backward_matches_fp64_autograd(dtype, has_bias, route):
    """DepthLayer's g_feat, g_weight and g_bias against fp64 autograd of F.conv2d on the same rounded operands (features in the
    type, weights rounded to it).  channels_last is the layout LiftTrainModel feeds; feature_input: the features need no gradient;
    frozen_weight: the weight needs none.  n_out = 128 makes a transposed (out, in) weight the same shape as the right one."""
    N, h, w = 2, 8, 17
    for n_out in (65, 128):
        torch.manual_seed(n_out + 3 * len(route))
        layer = DepthLayer(n_out, bias=has_bias).to(DEV)
        if route == "frozen_weight":
            layer.weight.requires_grad_(False)
        g = _gen(n_out)
        feat = torch.randn(N, 128, h, w, generator=g, device=DEV).to(dtype)
        if route == "channels_last":
            feat = feat.contiguous(memory_format=torch.channels_last)
        feat.requires_grad_(route != "feature_input")
        head = layer(feat)
        gout = torch.randn(head.shape, generator=g, device=DEV)
        head.backward(gout)

        x64 = feat.detach().double().requires_grad_(True)
        w64 = layer.weight.detach().to(dtype).double().requires_grad_(True)
        b64 = layer.bias.detach().double().requires_grad_(True) if has_bias else None
        F.conv2d(x64, w64, b64).backward(gout.double())
        u, what = UNIT[dtype], (route, n_out)
        g_abs = gout.double().abs()
        if route == "feature_input":
            assert feat.grad is None
        else:                                                 # sum over the n_out output channels
            assert feat.grad.dtype == dtype
            _assert_grad_bound(feat.grad, x64.grad, F.conv_transpose2d(g_abs, w64.detach().abs()), u, n_out, what + ("g_feat",))
        k = N * h * w                                         # sum over the images' pixels
        if route == "frozen_weight":
            assert layer.weight.grad is None
        else:
            assert layer.weight.grad.dtype == torch.float32
            terms = torch.einsum("nohw,nihw->oi", g_abs, x64.detach().abs()).view(n_out, 128, 1, 1)
            _assert_grad_bound(layer.weight.grad, w64.grad, terms, u, k, what + ("g_weight",))
        if has_bias:
            assert layer.bias.grad.dtype == torch.float32
            _assert_grad_bound(layer.bias.grad, b64.grad, g_abs.sum((0, 2, 3)), u, k, what + ("g_bias",))


# ==== C. first BEV convolution ===================================================================================================
def _conv_call(x_nhwc, pw, scale=None, shift=None, relu=False):
    """fiery_bev_first_conv_forward on a guarded output.  A CTA addresses rows oy < Ho + 7 and columns ox < Wo + 15 of its frame, so
    no store of the last frame, guarded or not, reaches (8 * Wo + 16) * 64 floats past the end: that is the margin."""
    B, H, W, _ = x_nhwc.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    n = B * Ho * Wo * 64
    buf = _guarded(n, (8 * Wo + 16) * 64)
    _lib.check(_lib.load().fiery_bev_first_conv_forward(B, H, W, x_nhwc.data_ptr(), pw.data_ptr(),
                                                        scale.data_ptr() if scale is not None else None,
                                                        shift.data_ptr() if shift is not None else None, 1 if relu else 0,
                                                        buf.data_ptr(), _stream()),
               "fiery_bev_first_conv_forward")
    _assert_written_and_contained(buf, n, (B, H, W))
    return buf[:n].view(B, Ho, Wo, 64)


# (H, W): Ho = ceil(H / 2) and Wo = ceil(W / 2) rows / columns of 8 x 16 output patches
CV_GRIDS = [(1, 1), (2, 3), (7, 7), (1, 40), (40, 1),       # the 7-tap window covers both borders of an axis at once
            (16, 32),                                       # one output patch, exactly
            (32, 64),                                       # exact multiples
            (29, 61), (33, 65),                             # the largest tails (Ho % 8 = 7, Wo % 16 = 15) and tails of 1
            (51, 49), (101, 99), (250, 200)]                # the lift envelope's grids


def test_first_conv_grids_cover_every_tail_class():
    ho = {((H - 1) // 2 + 1) % 8 for H, _ in CV_GRIDS}
    wo = {((W - 1) // 2 + 1) % 16 for _, W in CV_GRIDS}
    assert {0, 1, 7} <= ho and {0, 1, 15} <= wo, (ho, wo)
    single = [(H, W) for H, W in CV_GRIDS if (H - 1) // 2 + 1 <= 8 and (W - 1) // 2 + 1 <= 16]
    assert (16, 32) in single and len(single) == 4, single
    assert sum(1 for H, W in CV_GRIDS if min(H, W) <= 7) == 5       # one window covers both borders of an axis


def _epilogue(t, scale, shift, relu):
    if scale is not None:
        t = t * scale.double().view(1, 1, 1, -1) + shift.double().view(1, 1, 1, -1)
    return t.clamp_min(0) if relu else t


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H,W", CV_GRIDS, ids=[f"{h}x{w}" for h, w in CV_GRIDS])
def test_first_conv_integers_bit_exact_with_every_epilogue(H, W, B):
    """Small integers (|sum| < 2^24: exact in TF32 operands and fp32 accumulation) against the fp64 convolution, bit for bit: every
    tap's stride-2 coordinates, the zero fill on all four borders, the tail patches.  The epilogues use power-of-two scales and
    integer shifts, so the fmaf is exact; relu must clip something in each relu case."""
    g = _gen(H * 1000 + W + B)
    x = _ints((B, H, W, 64), -3, 3, g)
    w = _ints((64, 64, 7, 7), -2, 2, g)
    pw = pack_conv_weight(w)
    conv = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), stride=2, padding=3).permute(0, 2, 3, 1)
    scale = torch.where(_ints((64,), 0, 1, g) > 0, 1.0, -1.0).to(DEV) * torch.exp2(_ints((64,), -2, 2, g))
    shift = _ints((64,), -20, 20, g)
    for sc, sh, relu in ((None, None, False), (scale, shift, False), (None, None, True), (scale, shift, True)):
        want = _epilogue(conv, sc, sh, relu)
        if relu:
            assert bool((_epilogue(conv, sc, sh, False) < 0).any()) and bool((want > 0).any())
        got = _conv_call(x, pw, sc, sh, relu)
        assert torch.equal(got, want.float()), (sc is None, relu, float((got.double() - want).abs().max()))


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H,W", CV_GRIDS, ids=[f"{h}x{w}" for h, w in CV_GRIDS])
def test_first_conv_random_fp32_matches_fp64(H, W, B):
    """The bars of tests/test_bev_conv_gpu.py: 1e-3 normwise and 2e-3 of the output scale element-wise against fp64, and within 3x of
    a TF32 convolution.  On tiny maps cuDNN may pick an fp32 kernel even with TF32 allowed, so the TF32 error it is compared with is
    the larger of cuDNN's and that of an fp64 convolution of the operands rounded to TF32."""
    g = _gen(H * 7 + W * 13 + B)
    x = torch.randn(B, H, W, 64, generator=g, device=DEV).permute(0, 3, 1, 2)
    w = torch.randn(64, 64, 7, 7, generator=g, device=DEV) * 0.02
    got = first_conv_forward(x, pack_conv_weight(w))
    assert tuple(got.shape) == (B, 64, (H - 1) // 2 + 1, (W - 1) // 2 + 1) and got.permute(0, 2, 3, 1).is_contiguous()
    want = F.conv2d(x.double(), w.double(), stride=2, padding=3)
    e = _nerr(got, want)
    assert e < 1e-3, e
    assert float((got.double() - want).abs().max()) < 2e-3 * float(want.abs().max())
    torch.backends.cudnn.allow_tf32 = True
    try:
        e_cudnn = _nerr(F.conv2d(x, w, stride=2, padding=3), want)
    finally:
        torch.backends.cudnn.allow_tf32 = False
    e_rounded = _nerr(F.conv2d(_tf32(x).double(), _tf32(w).double(), stride=2, padding=3), want)
    assert e <= max(3 * max(e_cudnn, e_rounded), 5e-4), (e, e_cudnn, e_rounded)


def test_first_conv_writes_every_output_and_nothing_past_it():
    """51 x 49 -> 26 x 25: the last row of patches has 2 live rows of 8 and each row's last patch 9 live columns of 16; two frames,
    so a stray store of frame 0 lands in frame 1 and one of frame 1 in the margin.  Checked in _conv_call; values exact."""
    g = _gen(4)
    x = _ints((2, 51, 49, 64), -3, 3, g)
    w = _ints((64, 64, 7, 7), -2, 2, g)
    got = _conv_call(x, pack_conv_weight(w))
    assert torch.equal(got, F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), stride=2, padding=3).permute(0, 2, 3, 1).float())


def test_first_conv_contract_edges_and_conversions():
    from fiery_b200._lib import FieryError
    lib = _lib.load()
    g = _gen(9)
    x = _ints((2, 23, 30, 64), -3, 3, g)
    w = _ints((64, 64, 7, 7), -2, 2, g)
    pw = pack_conv_weight(w)
    out = torch.full((2 * 12 * 15 * 64,), SENTINEL, device=DEV)
    _lib.check(lib.fiery_bev_first_conv_forward(0, 23, 30, x.data_ptr(), pw.data_ptr(), None, None, 0, out.data_ptr(), _stream()),
               "no frames")
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all())
    scale = torch.ones(64, device=DEV)
    with pytest.raises(FieryError, match="scale and shift go together"):
        _lib.check(lib.fiery_bev_first_conv_forward(2, 23, 30, x.data_ptr(), pw.data_ptr(), scale.data_ptr(), None, 0, out.data_ptr(),
                                                    _stream()), "scale without shift")
    with pytest.raises(FieryError, match="scale and shift go together"):
        first_conv_forward(x.permute(0, 3, 1, 2), pw, scale=scale)
    want = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), stride=2, padding=3).float()
    nchw = x.permute(0, 3, 1, 2).contiguous()                 # NCHW strides: converted to channels-last first
    assert nchw.is_contiguous() and not nchw.permute(0, 2, 3, 1).is_contiguous()
    assert torch.equal(first_conv_forward(nchw, pw).contiguous(), want)
    half = x.permute(0, 3, 1, 2).half()                       # fp16 input: widened first (small integers are exact)
    got = first_conv_forward(half, pw)
    assert got.dtype == torch.float32 and torch.equal(got.contiguous(), want)


# ==== D. the training step's gradient ============================================================================================
TRAIN_CFG = LiftConfig(**{**CONFIGS["cfg1_tiny"].__dict__})
# The step runs in fp32 except the depth layer's forward, which multiplies TF32 operands: its head is within 1e-3 normwise of fp64
# (the TF32 bar of the depth-layer tests).  Everything after it -- softmax, pooling, the BEV head, the loss and their gradients, and
# the fp32 backward of the depth layer (TF32 off here) -- is a smooth function of the head whose fp32 evaluation adds ~1e-6.  A
# relative perturbation of 1e-3 in the head moves the loss by at most the same order and each parameter's gradient by its
# condition number times 1e-3; the chain (softmax, sums, 1x1 / 3x3 convolutions, sigmoid, CE / L2 / L1) has no large one, and 10x
# covers it: gradients to 1e-2 normwise per parameter, the loss to 1e-3.  A gradient from a wrong layout or wrong weights is off by
# O(1).
TRAIN_GRAD_TOL, TRAIN_LOSS_TOL = 1e-2, 1e-3


def _replica_loss_and_grads(model, batch, feature_input, cfg):
    """The same model in fp64 on the CPU: the parameters copied, the depth layer as F.conv2d, the lift as direct fp64 pooling at the
    oracle's voxel indices (like _oracle_grad(exact=True) in tests/test_lift_backward_gpu.py), the BEV head and the loss of
    LiftTrainModel.  Returns the loss and every trainable parameter's gradient by name."""
    P = {n: p.detach().cpu().double().requires_grad_(True) for n, p in model.named_parameters() if p.requires_grad}
    image = batch["image"].cpu().double()
    b, s, n = image.shape[:3]
    x = image.reshape(b * s * n, *image.shape[3:])
    if not feature_input:
        for i in (0, 2, 4):
            x = F.relu(F.conv2d(x, P[f"encoder.features.{i}.weight"], P[f"encoder.features.{i}.bias"], stride=2, padding=1))
    head = F.conv2d(x, P["encoder.depth_layer.weight"], P["encoder.depth_layer.bias"])
    oracle = O.LiftOracle.from_config(cfg)
    K = batch["intrinsics"].cpu().reshape(b * s, n, 3, 3)
    E = batch["extrinsics"].cpu().reshape(b * s, n, 4, 4)
    idx, keep = oracle.point_indices(K, E)
    vol = O.depth_context_volume(head, n, oracle.D, oracle.C, oracle.use_depth_distribution)
    X, Y = cfg.bev_hw
    C = oracle.C
    frames = []
    for f in range(b * s):
        cell = idx[f][keep[f]]
        frames.append(torch.zeros(X * Y, C, dtype=torch.float64).index_add(0, cell[:, 0] * Y + cell[:, 1], vol[f].reshape(-1, C)[keep[f]]))
    bev = torch.stack(frames).view(b * s, X, Y, C).permute(0, 3, 1, 2)
    t = F.relu(F.conv2d(bev, P["head.trunk.0.weight"], P["head.trunk.0.bias"], padding=1))
    seg = F.conv2d(t, P["head.segmentation.weight"], P["head.segmentation.bias"])
    cen = torch.sigmoid(F.conv2d(t, P["head.centerness.weight"], P["head.centerness.bias"]))
    off = F.conv2d(t, P["head.offset.weight"], P["head.offset.bias"])
    l_seg = F.cross_entropy(seg, batch["segmentation"].cpu().reshape(b * s, X, Y))
    l_cen = F.mse_loss(cen, batch["centerness"].cpu().double().reshape(b * s, 1, X, Y))
    l_off = F.l1_loss(off, batch["offset"].cpu().double().reshape(b * s, 2, X, Y))
    ws, wc, wo = P["segmentation_weight"], P["centerness_weight"], P["offset_weight"]
    loss = (l_seg / torch.exp(ws) + 0.5 * ws + l_cen / (2 * torch.exp(wc)) + 0.5 * wc + l_off / (2 * torch.exp(wo)) + 0.5 * wo)
    loss.backward()
    return float(loss.detach()), {k: v.grad for k, v in P.items()}        # None: a parameter the step does not use


@pytest.mark.parametrize("feature_input", [True, False], ids=["features", "images"])
def test_training_step_gradient_matches_fp64_replica(feature_input):
    tr = LiftTrainer(TRAIN_CFG, DEV, precision=32, feature_input=feature_input, seed=3)
    batch = synthetic_batch(TRAIN_CFG, 2, 2, DEV, seed=9, feature_input=feature_input)
    loss = float(tr.forward_backward(batch))
    flat = tr.bucket.flat.detach().cpu()
    want_loss, want = _replica_loss_and_grads(tr.model, batch, feature_input, TRAIN_CFG)
    assert abs(loss - want_loss) <= TRAIN_LOSS_TOL * abs(want_loss), (loss, want_loss)
    named = [(k, p) for k, p in tr.model.named_parameters() if p.requires_grad]
    assert len(named) == len(tr.bucket.params) and all(p is q for (_, p), q in zip(named, tr.bucket.params))
    assert set(want) == {k for k, _ in named}
    off = 0
    for k, p in named:                                        # the bucket's order
        got = flat[off:off + p.numel()].view(p.shape)
        off += p.numel()
        if want[k] is None:                                   # the image encoder when the step starts from features
            assert feature_input and k.startswith("encoder.features") and float(got.abs().max()) == 0, k
            continue
        assert float(want[k].norm()) > 0, k
        assert O.normwise_error(got, want[k]) < TRAIN_GRAD_TOL, (k, O.normwise_error(got, want[k]))
    assert off == flat.numel()
