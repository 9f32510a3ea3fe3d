"""GPU: the wgmma first BEV convolution (fiery_b200/csrc/bev_conv.cu; Decoder.first_conv + bn1 + relu, fiery/models/decoder.py:11,
59-61) against torch convolutions of the same layer.

Parity bar: the kernel multiplies TF32 operands (10-bit mantissa; weights rounded at packing time, activations truncated by the
tensor core) and accumulates in fp32 -- the precision cuDNN uses for this layer under torch's default ``cudnn.allow_tf32``.  Against
an fp64 convolution the bar is 1e-3 normwise and 2e-3 of the output scale element-wise (a 3136-term TF32 dot product: 3e-4 with both
operands rounded, ~7e-4 with truncated activations), and the kernel must stay within 3x of cuDNN's own TF32 result on the same
inputs."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fiery_b200.bev_conv import FirstConv, first_conv_forward, pack_weight

pytestmark = pytest.mark.gpu


def _nerr(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("B,H,W", [(1, 200, 200), (3, 200, 200), (2, 400, 200), (1, 50, 50), (2, 37, 61)])
def test_first_conv_matches_fp64_convolution(B, H, W):
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(B * 1000 + H + W)
    x = torch.randn(B, H, W, 64, generator=g).to(dev).permute(0, 3, 1, 2)           # channels-last strides, as the lift returns it
    w = (torch.randn(64, 64, 7, 7, generator=g) * 0.02).to(dev)
    got = first_conv_forward(x, pack_weight(w))
    assert tuple(got.shape) == (B, 64, (H - 1) // 2 + 1, (W - 1) // 2 + 1) and got.dtype == torch.float32
    assert got.permute(0, 2, 3, 1).is_contiguous()
    want = F.conv2d(x.double(), w.double(), stride=2, padding=3)
    e = _nerr(got, want)
    assert e < 1e-3, e
    assert float((got.double() - want).abs().max()) < 2e-3 * float(want.abs().max())
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        e_cudnn = _nerr(F.conv2d(x, w, stride=2, padding=3), want)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    assert e <= max(3 * e_cudnn, 5e-4), (e, e_cudnn)


def test_borders_and_packing_are_exact_on_integers():
    """Small integers are exact in TF32 and fp32: the result must equal the fp32 convolution BIT FOR BIT -- checks the im2col
    coordinates, the zero padding on all four borders, the tap order of the packed weights and the accumulator -> pixel mapping."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(7)
    x = torch.randint(-3, 4, (2, 45, 83, 64), generator=g).float().to(dev).permute(0, 3, 1, 2)
    w = torch.randint(-2, 3, (64, 64, 7, 7), generator=g).float().to(dev)
    got = first_conv_forward(x, pack_weight(w))
    want = F.conv2d(x.double(), w.double(), stride=2, padding=3).float()
    assert torch.equal(got.contiguous(), want)
    p = pack_weight(w)
    assert torch.equal(p, w.permute(2, 3, 0, 1).reshape(49, 64, 64))      # small integers are TF32 numbers: rounding keeps them


def test_module_folds_bn_relu_like_the_decoder():
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    conv = torch.nn.Conv2d(64, 64, kernel_size=7, stride=2, padding=3, bias=False).to(dev)
    bn = torch.nn.BatchNorm2d(64).to(dev)
    with torch.no_grad():
        bn.running_mean.normal_(0, 0.1)
        bn.running_var.uniform_(0.5, 2.0)
        bn.weight.normal_(1.0, 0.1)
        bn.bias.normal_(0, 0.1)
    import types
    dec = types.SimpleNamespace(first_conv=conv, bn1=bn)
    m = FirstConv.from_decoder(dec).eval()
    assert m.weight is conv.weight
    x = torch.randn(2, 100, 100, 64, device=dev).permute(0, 3, 1, 2)
    bn.eval()
    with torch.no_grad():
        want = torch.relu(bn(conv(x.double().float()))).double()
        want64 = torch.relu(F.batch_norm(F.conv2d(x.double(), conv.weight.double(), stride=2, padding=3), bn.running_mean.double(),
                                         bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps))
    got = m(x)
    assert _nerr(got, want64) < 1e-3
    assert float((got < 0).sum()) == 0
    with torch.no_grad():
        conv.weight.mul_(2.0)                                   # in-place update: the packed copy follows the parameter's version
    assert _nerr(m(x), torch.relu(F.batch_norm(F.conv2d(x.double(), conv.weight.double(), stride=2, padding=3), bn.running_mean.double(),
                                               bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps))) < 1e-3
    with pytest.raises(RuntimeError):
        m.train()(x)


def test_lift_to_first_conv_without_a_layout_pass():
    """The lift's channel-last BEV feeds the convolution directly (no NCHW pass in between)."""
    from fiery_b200.lift import LiftSplat
    from fiery_b200.synthetic import CONFIGS, LiftConfig, make_calibration, make_head
    cfg = LiftConfig(**{**CONFIGS["cfg2_static_lss"].__dict__, "frames": 2})
    dev = torch.device("cuda:0")
    K, E = make_calibration(cfg, seed=5)
    lift = LiftSplat.from_config(cfg, output_layout="channels_last").to(dev)
    with torch.no_grad():
        bev = lift(torch.from_numpy(make_head(cfg, seed=5)).to(dev), torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev))
    assert bev.permute(0, 2, 3, 1).is_contiguous()
    w = (torch.randn(64, 64, 7, 7, device=dev) * 0.02)
    got = first_conv_forward(bev, pack_weight(w))
    want = F.conv2d(bev.double(), w.double(), stride=2, padding=3)
    assert _nerr(got, want) < 1e-3
