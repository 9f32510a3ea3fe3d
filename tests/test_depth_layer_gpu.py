"""GPU: Encoder.depth_layer (fiery/models/encoder.py:36,96) as a wgmma GEMM writing the fp32 head tensor
(fiery_b200/csrc/depth_layer.cu).  Parity bar: fp16 / bf16 / TF32 operands with fp32 accumulation -- what cuDNN does for this layer
under autocast / allow_tf32 -- against an fp64 convolution of the SAME rounded operands: 1e-5 normwise (only the fp32 accumulation
order differs), and against the unrounded fp64 convolution: 2e-3 (fp16), 1e-2 (bf16), 1e-3 (TF32)."""
import pytest
import torch
import torch.nn.functional as F

from fiery_b200.depth_layer import DepthLayer, depth_layer_forward

pytestmark = pytest.mark.gpu


def _nerr(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("dtype,tol", [(torch.float16, 2e-3), (torch.bfloat16, 1e-2), (torch.float32, 1e-3)])
@pytest.mark.parametrize("N,h,w,n_out", [(6, 28, 60, 112), (2, 8, 16, 112), (3, 28, 60, 64), (1, 5, 16, 100)])
def test_depth_layer_matches_convolution(dtype, tol, N, h, w, n_out):
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(N * 100 + h + n_out)
    feat = torch.randn(N, 128, h, w, generator=g).to(dev).to(dtype)
    weight = (torch.randn(n_out, 128, 1, 1, generator=g) * 0.1).to(dev)
    bias = torch.randn(n_out, generator=g).to(dev)
    got = depth_layer_forward(feat, weight, bias)
    assert tuple(got.shape) == (N, n_out, h, w) and got.dtype == torch.float32 and got.is_contiguous()
    exact = F.conv2d(feat.double(), weight.double(), bias.double())
    assert _nerr(got, exact) < tol
    if dtype != torch.float32:                              # same rounded operands, exact products: only the summation order differs
        same = F.conv2d(feat.double(), weight.to(dtype).double(), bias.double())
        assert _nerr(got, same) < 1e-5
    assert float(depth_layer_forward(feat, weight, None).sub(got).add(bias.view(1, -1, 1, 1)).abs().max()) < 1e-5


def test_small_integers_are_exact():
    """Integers are exact in every operand type: bit-equality with the fp32 convolution checks the operand layouts (K-major weights,
    pixel-contiguous features), the tile / image / channel addressing and the ragged last tile of an image.  40 images = 560 tiles:
    every persistent CTA runs several tiles, so the feature ring and both accumulators wrap."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(1)
    for dtype in (torch.float16, torch.float32):
        feat = torch.randint(-4, 5, (40, 128, 28, 60), generator=g).float().to(dev).to(dtype)
        weight = torch.randint(-3, 4, (112, 128, 1, 1), generator=g).float().to(dev)
        bias = torch.randint(-8, 9, (112,), generator=g).float().to(dev)
        assert torch.equal(depth_layer_forward(feat, weight, bias), F.conv2d(feat.float(), weight, bias))


def test_unsupported_row_pitch_is_an_error_not_a_fallback():
    from fiery_b200._lib import FieryError
    feat = torch.randn(1, 128, 5, 12, device="cuda:0").half()              # 60 pixels x 2 bytes: not a 16-byte pitch (TMA)
    with pytest.raises(FieryError, match="16-byte row pitch"):
        depth_layer_forward(feat, torch.randn(112, 128, 1, 1, device="cuda:0"), None)
    with pytest.raises(Exception):
        depth_layer_forward(feat.cpu(), torch.randn(112, 128, 1, 1), None)


def test_packed_weights_follow_the_parameter():
    dev = torch.device("cuda:0")
    layer = DepthLayer(112).to(dev)
    feat = torch.randn(2, 128, 8, 16, device=dev).half()
    a = layer(feat)
    with torch.no_grad():
        layer.weight.mul_(2.0)                                              # an optimizer step bumps the version
    b = layer(feat)
    want = F.conv2d(feat.double(), layer.weight.half().double(), layer.bias.double())
    assert _nerr(b, want) < 1e-5 and _nerr(a, want) > 0.1


def test_module_is_a_drop_in_with_gradients_and_feeds_the_lift():
    from fiery_b200.lift import LiftSplat
    from fiery_b200.synthetic import CONFIGS, LiftConfig, make_calibration
    from oracle import lift_oracle as O
    cfg = LiftConfig(**{**CONFIGS["cfg1_tiny"].__dict__, "frames": 2})
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(128, cfg.head_channels, kernel_size=1, padding=0).to(dev)
    layer = DepthLayer.from_conv(conv)
    assert layer.weight is conv.weight and layer.bias is conv.bias and set(layer.state_dict()) == set(conv.state_dict())
    h, w = cfg.feat_hw
    feat = torch.randn(cfg.frames * cfg.n_cameras, 128, h, w, device=dev).half().requires_grad_(True)
    K, E = make_calibration(cfg, seed=4)
    Kd, Ed = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
    lift = LiftSplat.from_config(cfg).to(dev)
    head = layer(feat)                                       # fp16 features in, fp32 head out: no widening pass before the lift
    assert head.dtype == torch.float32
    bev = lift(head, Kd, Ed)
    bev.square().sum().backward()
    g_feat, g_w, g_b = feat.grad.clone(), conv.weight.grad.clone(), conv.bias.grad.clone()
    # the same graph with torch's convolution in fp32 on the same rounded features
    feat2 = feat.detach().float().requires_grad_(True)
    conv.zero_grad()
    w16 = conv.weight.to(torch.float16).float()
    head2 = F.conv2d(feat2, w16, conv.bias)
    assert _nerr(head, head2) < 1e-5
    lift(head2, Kd, Ed).square().sum().backward()
    assert _nerr(g_feat, feat2.grad) < 2e-3                  # fp16 gradient of the features
    exact = O.LiftOracle.from_config(cfg).lift_exact(head.detach().cpu(), torch.from_numpy(K), torch.from_numpy(E))
    assert O.normwise_error(bev.detach().cpu(), exact) < 1e-4
    assert g_w.shape == conv.weight.shape and g_b.shape == conv.bias.shape and float(g_w.abs().sum()) > 0
