"""GPU: the backward of the first BEV convolution (fiery_b200/csrc/bev_conv_bwd.cu: input and weight gradients of Decoder.first_conv,
fiery/models/decoder.py:11,59) and the ``fiery_b200::first_conv`` operator / ``FirstConv`` module that train through it.

Parity bar (the forward's, tests/test_bev_conv_gpu.py): TF32 operands and fp32 accumulation against fp64 autograd of F.conv2d --
normwise < 1e-3, element-wise < 2e-3 of the gradient's scale, and within 3x of the larger of cuDNN TF32's backward error and the
error of the fp64 backward on TF32-rounded operands.  Small integers are exact in TF32 and fp32, so on them both gradients must be
bit-exact."""
import ctypes
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from fiery_b200 import _lib
from fiery_b200 import ops  # noqa: F401  (registers the operators)
from fiery_b200.bev_conv import (FirstConv, backward_weight_workspace_bytes, first_conv_backward_data, first_conv_backward_weight,
                                 pack_weight_transposed)

pytestmark = pytest.mark.gpu

GRIDS = [(1, 1), (2, 3), (7, 7), (1, 40), (40, 1), (16, 32), (32, 64), (29, 61), (33, 65), (51, 49), (101, 99), (250, 200)]
MARGIN = 4096                                   # sentinel floats after every output


@pytest.fixture(autouse=True, scope="module")
def _no_tf32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _dev():
    return torch.device("cuda:0")


def _nerr(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _tf32(t):
    """fp32 -> TF32, round to nearest, ties away from zero (cvt.rna), as an fp32 tensor."""
    b = t.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def _ho(n):
    return (n - 1) // 2 + 1


def _fp64_grads(x, w, gy):
    x64 = x.detach().double().requires_grad_(True)
    w64 = w.detach().double().requires_grad_(True)
    F.conv2d(x64, w64, stride=2, padding=3).backward(gy.detach().double())
    return x64.grad, w64.grad


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _raw_dgrad(gy_nhwc, pt, B, H, W):
    """fiery_bev_first_conv_backward_data into a NaN-filled buffer with a NaN sentinel margin; returns (grad_x NHWC, margin)."""
    n = B * H * W * 64
    buf = torch.full((n + MARGIN,), float("nan"), device=_dev())
    _lib.check(_lib.load().fiery_bev_first_conv_backward_data(B, H, W, gy_nhwc.data_ptr(), pt.data_ptr(), buf.data_ptr(), _stream()),
               "dgrad")
    return buf[:n].view(B, H, W, 64), buf[n:]


def _raw_wgrad(x_nhwc, gy_nhwc, B, H, W, ws_fill=float("nan")):
    nbytes = backward_weight_workspace_bytes(B, H, W)
    ws = torch.full((max(nbytes // 4, 4),), ws_fill, device=_dev())
    n = 64 * 64 * 49
    buf = torch.full((n + MARGIN,), float("nan"), device=_dev())
    _lib.check(_lib.load().fiery_bev_first_conv_backward_weight(B, H, W, x_nhwc.data_ptr() if x_nhwc is not None else None,
                                                                gy_nhwc.data_ptr() if gy_nhwc is not None else None, buf.data_ptr(),
                                                                ws.data_ptr(), _stream()), "wgrad")
    return buf[:n].view(64, 64, 7, 7), buf[n:]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H,W", GRIDS)
def test_small_integers_are_bit_exact(B, H, W):
    g = torch.Generator(device="cpu").manual_seed(B * 7919 + H * 131 + W)
    x = torch.randint(-3, 4, (B, H, W, 64), generator=g).float().to(_dev())
    gy = torch.randint(-2, 3, (B, _ho(H), _ho(W), 64), generator=g).float().to(_dev())
    w = torch.randint(-2, 3, (64, 64, 7, 7), generator=g).float().to(_dev())
    want_x, want_w = _fp64_grads(x.permute(0, 3, 1, 2), w, gy.permute(0, 3, 1, 2))
    gx, margin = _raw_dgrad(gy, pack_weight_transposed(w), B, H, W)
    assert not torch.isnan(gx).any() and torch.isnan(margin).all()
    assert torch.equal(gx.permute(0, 3, 1, 2).double(), want_x)
    gw, margin = _raw_wgrad(x, gy, B, H, W)
    assert not torch.isnan(gw).any() and torch.isnan(margin).all()
    assert torch.equal(gw.double(), want_w)


def test_transposed_pack_layout_and_rounding():
    w = torch.randn(64, 64, 7, 7, device=_dev())
    pt = pack_weight_transposed(w)
    assert torch.equal(pt, _tf32(w.permute(2, 3, 1, 0).reshape(49, 64, 64)))


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H,W", GRIDS)
def test_random_fp32_within_the_tf32_bar(B, H, W):
    g = torch.Generator(device="cpu").manual_seed(B * 104729 + H * 37 + W)
    x = torch.randn(B, H, W, 64, generator=g).to(_dev()).permute(0, 3, 1, 2)
    gy = torch.randn(B, _ho(H), _ho(W), 64, generator=g).to(_dev()).permute(0, 3, 1, 2)
    w = (torch.randn(64, 64, 7, 7, generator=g) * 0.02).to(_dev())
    want_x, want_w = _fp64_grads(x, w, gy)
    got_x = first_conv_backward_data(gy, pack_weight_transposed(w), H, W)
    got_w = first_conv_backward_weight(x, gy)
    assert got_x.permute(0, 2, 3, 1).is_contiguous() and got_x.dtype == torch.float32
    # the two references: cuDNN's TF32 backward, and the fp64 backward of TF32-rounded operands
    torch.backends.cudnn.allow_tf32 = True
    try:
        cx, cw, _ = torch.ops.aten.convolution_backward(gy, x, w, None, [2, 2], [3, 3], [1, 1], False, [0, 0], 1, [True, True, False])
    finally:
        torch.backends.cudnn.allow_tf32 = False
    rx, rw = _fp64_grads(_tf32(x), _tf32(w), _tf32(gy))
    for got, want, cud, rnd in ((got_x, want_x, cx, rx), (got_w, want_w, cw, rw)):
        e = _nerr(got, want)
        assert e < 1e-3, e
        assert float((got.double() - want).abs().max()) < 2e-3 * float(want.abs().max())
        bar = max(_nerr(cud, want), _nerr(rnd, want))
        assert e <= 3 * bar, (e, bar)


def test_gradients_are_reproducible_eager_and_in_a_graph():
    B, H, W = 2, 101, 99
    g = torch.Generator(device="cpu").manual_seed(11)
    x = torch.randn(B, H, W, 64, generator=g).to(_dev())
    gy = torch.randn(B, _ho(H), _ho(W), 64, generator=g).to(_dev())
    w = torch.randn(64, 64, 7, 7, generator=g).to(_dev()) * 0.02
    pt = pack_weight_transposed(w)
    runs = []
    for fill in (float("nan"), 1e30, 0.0):
        gx, _ = _raw_dgrad(gy, pt, B, H, W)
        gw, _ = _raw_wgrad(x, gy, B, H, W, ws_fill=fill)
        runs.append((gx.clone(), gw.clone()))
    for gx, gw in runs[1:]:
        assert torch.equal(gx, runs[0][0]) and torch.equal(gw, runs[0][1])
    xc, gyc = x.permute(0, 3, 1, 2), gy.permute(0, 3, 1, 2)
    ws = torch.full((backward_weight_workspace_bytes(B, H, W),), 255, dtype=torch.uint8, device=_dev())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        first_conv_backward_data(gyc, pt, H, W)
        first_conv_backward_weight(xc, gyc, ws)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_x = first_conv_backward_data(gyc, pt, H, W)
        out_w = first_conv_backward_weight(xc, gyc, ws)
    for fill in (0, 7, 255):
        ws.fill_(fill)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out_x.permute(0, 2, 3, 1), runs[0][0]) and torch.equal(out_w, runs[0][1])


def test_no_frames_gives_zero_weight_gradient():
    gw, margin = _raw_wgrad(None, None, 0, 200, 200)
    assert torch.equal(gw, torch.zeros_like(gw)) and torch.isnan(margin).all()
    x = torch.empty(0, 64, 20, 20, device=_dev())
    gy = torch.empty(0, 64, 10, 10, device=_dev())
    assert torch.equal(first_conv_backward_weight(x, gy), torch.zeros(64, 64, 7, 7, device=_dev()))
    assert first_conv_backward_data(gy, pack_weight_transposed(torch.randn(64, 64, 7, 7, device=_dev())), 20, 20).shape == (0, 64, 20, 20)


def test_operator_backward_takes_nchw_grad_and_half_input():
    torch.manual_seed(5)
    x = torch.randn(2, 64, 33, 65, device=_dev())
    w = torch.randn(64, 64, 7, 7, device=_dev()) * 0.02
    gy_cl = torch.randn(2, 17, 33, 64, device=_dev()).permute(0, 3, 1, 2)
    gx1, gw1 = torch.ops.fiery_b200.first_conv_backward(gy_cl, x, w, True, True)
    gx2, gw2 = torch.ops.fiery_b200.first_conv_backward(gy_cl.contiguous(), x, w, True, True)      # NCHW-contiguous grad_y
    assert torch.equal(gx1, gx2) and torch.equal(gw1, gw2)
    assert gx1.permute(0, 2, 3, 1).is_contiguous() and gx1.dtype == torch.float32
    xh = x.half().requires_grad_(True)
    wp = w.clone().requires_grad_(True)
    y = torch.ops.fiery_b200.first_conv(xh, wp)
    assert y.dtype == torch.float32
    y.backward(gy_cl)
    assert xh.grad.dtype == torch.float16 and xh.grad.shape == xh.shape
    want_x, want_w = _fp64_grads(xh.detach().float(), w, gy_cl)
    assert _nerr(xh.grad, want_x) < 1.5e-3 and _nerr(wp.grad, want_w) < 1e-3


def _reference_conv(weight):
    conv = nn.Conv2d(64, 64, 7, 2, 3, bias=False).to(_dev())
    with torch.no_grad():
        conv.weight.copy_(weight)
    return conv


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("train", [False, True])
def test_first_conv_module_gradients(relu, train):
    torch.manual_seed(int(relu) * 2 + int(train))
    m = FirstConv(relu=relu).to(_dev()).train(train)
    x = torch.randn(2, 100, 98, 64, device=_dev()).permute(0, 3, 1, 2).requires_grad_(True)
    y = m(x)
    assert y.grad_fn is not None
    r = torch.randn_like(y)
    (y * r).sum().backward()
    x64 = x.detach().double().requires_grad_(True)
    w64 = m.weight.detach().double().requires_grad_(True)
    y64 = F.conv2d(x64, w64, stride=2, padding=3)
    if relu:
        # the relu's mask is taken from the module's own output: a TF32 rounding can flip the sign of an output near zero, and
        # the gradient of such an element is then legitimately 0 on one side and not on the other
        assert _nerr(y, torch.relu(y64)) < 1e-3
        y64 = y64 * (y.detach() > 0).double()
    else:
        assert _nerr(y, y64) < 1e-3
    (y64 * r.double()).sum().backward()
    assert _nerr(x.grad, x64.grad) < 1e-3 and _nerr(m.weight.grad, w64.grad) < 1e-3
    with torch.no_grad():                              # grad disabled: the fused inference kernel, same values
        assert torch.equal(m(x), y.detach())


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


def test_unneeded_gradients_are_not_launched():
    m = FirstConv().to(_dev())
    x = torch.randn(1, 64, 64, 64, device=_dev()).contiguous(memory_format=torch.channels_last)
    m(x.requires_grad_(True)).sum().backward()        # warm up: packs made once for this weight version
    m.weight.requires_grad_(False)
    names = _kernels(lambda: m(x).sum().backward())
    assert any("dgrad" in n for n in names) and not any("wgrad" in n for n in names)
    assert not any("pack_conv_weights" in n for n in names)           # cached per weight version
    m.weight.requires_grad_(True)
    x2 = x.detach()
    names = _kernels(lambda: m(x2).sum().backward())
    assert any("wgrad" in n for n in names) and not any("dgrad" in n for n in names)


def test_first_conv_under_autocast_and_compile():
    torch.manual_seed(9)
    m = FirstConv().to(_dev())
    x = torch.randn(2, 64, 60, 50, device=_dev()).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16):
        y = m(x)
    assert y.dtype == torch.float32                    # the operator runs in fp32 under AMP
    y.square().sum().backward()
    gx, gw = x.grad.clone(), m.weight.grad.clone()
    x64 = x.detach().double().requires_grad_(True)
    w64 = m.weight.detach().double().requires_grad_(True)
    F.conv2d(x64, w64, stride=2, padding=3).square().sum().backward()
    assert _nerr(gx, x64.grad) < 2e-3 and _nerr(gw, w64.grad) < 2e-3
    x.grad = None
    m.weight.grad = None
    step = torch.compile(lambda t: m(t).square().sum(), backend="aot_eager", fullgraph=True)
    step(x).backward()
    assert _nerr(x.grad, gx) < 1e-6 and _nerr(m.weight.grad, gw) < 1e-6


def _chain(cfg, conv_layer, seed=0):
    from fiery_b200.depth_layer import DepthLayer
    from fiery_b200.lift import LiftSplat
    from fiery_b200.synthetic import make_calibration
    dev = _dev()
    torch.manual_seed(seed)
    depth_conv = nn.Conv2d(128, cfg.head_channels, kernel_size=1).to(dev)
    layer = DepthLayer.from_conv(depth_conv)
    lift = LiftSplat.from_config(cfg, output_layout="channels_last").to(dev)
    bn = nn.BatchNorm2d(64).to(dev).train()
    h, w = cfg.feat_hw
    feat = torch.randn(cfg.frames * cfg.n_cameras, 128, h, w, device=dev)
    K, E = make_calibration(cfg, seed=seed)
    Kd, Ed = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
    seen = []
    orig = lift._launch_backward

    def spy(*a, **k):
        g = a[3]
        seen.append(g.permute(0, 2, 3, 1).is_contiguous() and not g.is_contiguous())
        return orig(*a, **k)
    lift._launch_backward = spy

    def run(mask=None):
        """Gradients of the chain; ``mask`` replaces the relu by a product with a fixed 0/1 mask (see the test)."""
        for p in (depth_conv.weight, depth_conv.bias, conv_layer.weight, bn.weight, bn.bias):
            p.grad = None
        head = layer(feat)
        head.retain_grad()
        pre = bn(conv_layer(lift(head, Kd, Ed)))
        out = torch.relu(pre) if mask is None else pre * mask
        r = torch.linspace(-1, 1, out.numel(), device=dev).view(out.shape)
        (out * r).sum().backward()
        return [head.grad.clone(), depth_conv.weight.grad.clone(), conv_layer.weight.grad.clone()], (pre > 0).detach()
    return run, seen


def test_chain_depth_layer_lift_first_conv_bn_relu():
    from fiery_b200.synthetic import CONFIGS, LiftConfig
    cfg = LiftConfig(**{**CONFIGS["cfg1_tiny"].__dict__, "frames": 2})
    torch.manual_seed(1)
    ref_conv = nn.Conv2d(64, 64, 7, 2, 3, bias=False).to(_dev())
    ours = FirstConv.from_conv(copy.deepcopy(ref_conv))
    run_ref, _ = _chain(cfg, ref_conv)
    run_ours, seen = _chain(cfg, ours)
    got, mask = run_ours()
    # the reference chain takes the relu's mask from ours: TF32 rounding can flip the sign of a normalised value near zero, and that
    # element's gradient is then legitimately 0 on one side only
    want, _ = run_ref(mask.float())
    assert seen and all(seen)                          # the lift's backward got a channels-last gradient: its NHWC route
    for a, b in zip(got, want):
        assert _nerr(a, b) < 2e-3, _nerr(a, b)
    torch.use_deterministic_algorithms(True)
    try:
        runs = [run_ours()[0] for _ in range(3)]
    finally:
        torch.use_deterministic_algorithms(False)
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert torch.equal(a, b)


def test_use_tensor_core_first_conv_on_a_decoder():
    from fiery_b200.install import use_tensor_core_first_conv

    class Decoder(nn.Module):
        def __init__(self):
            super().__init__()
            self.first_conv = nn.Conv2d(64, 64, kernel_size=7, stride=2, padding=3, bias=False)
            self.bn1 = nn.BatchNorm2d(64)
            self.relu = nn.ReLU(inplace=True)

        def forward(self, x):
            return self.relu(self.bn1(self.first_conv(x)))

    class Model(nn.Module):
        def __init__(self):
            super().__init__()
            self.decoder = Decoder()

    torch.manual_seed(4)
    ref = Model().to(_dev())
    model = copy.deepcopy(ref)
    use_tensor_core_first_conv(model)
    assert isinstance(model.decoder.first_conv, FirstConv)
    x = torch.randn(2, 80, 90, 64, device=_dev()).permute(0, 3, 1, 2)
    outs = []
    mask = None
    for m in (model, ref):
        xi = x.clone().requires_grad_(True)
        pre = m.decoder.bn1(m.decoder.first_conv(xi))
        if mask is None:                               # ours: the decoder's own relu; the reference takes its mask (see the chain test)
            y = m.decoder.relu(pre)
            mask = (pre > 0).detach().float()
        else:
            y = pre * mask
        (y * torch.linspace(-1, 1, y.numel(), device=_dev()).view(y.shape)).sum().backward()
        outs.append((torch.relu(pre).detach(), xi.grad, m.decoder.first_conv.weight.grad.clone()))
    for a, b in zip(outs[0], outs[1]):
        assert _nerr(a, b) < 2e-3, _nerr(a, b)
    w = model.decoder.first_conv.weight
    before = w.detach().clone()
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    opt.step()
    assert not torch.equal(w.detach(), before)
    assert model.state_dict()["decoder.first_conv.weight"].data_ptr() == w.data_ptr()
    with torch.no_grad():                              # the forward follows the updated weight (packs re-made for the new version)
        want = F.conv2d(x.double(), w.double(), stride=2, padding=3)
        assert _nerr(model.decoder.first_conv(x), want) < 1e-3
