"""Time Encoder.depth_layer (1x1 conv 128 -> 112) on the wgmma kernel against cuDNN (+ the widening pass an AMP step needs)."""
import sys
import torch
import torch.nn.functional as F
from fiery_b200.depth_layer import depth_layer_forward, pack_weight

dev = torch.device("cuda:0")
frames = int(sys.argv[1]) if len(sys.argv) > 1 else 8
N, h, w, n_out = frames * 6, 28, 60, 112
flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, iters=30):
    for _ in range(5):
        fn()
    evs = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); evs.append((a, b))
    torch.cuda.synchronize()
    t = sorted(x.elapsed_time(y) for x, y in evs)
    return t[len(t) // 2] * 1e3


only = sys.argv[2] if len(sys.argv) > 2 else None
for dtype in ((torch.float16,) if only == 'fp16' else (torch.float16, torch.bfloat16, torch.float32)):
    feat = torch.randn(N, 128, h, w, device=dev).to(dtype)
    weight = torch.randn(n_out, 128, 1, 1, device=dev) * 0.1
    bias = torch.randn(n_out, device=dev)
    wd = weight.to(dtype)
    bd = bias.to(dtype)
    torch.backends.cudnn.allow_tf32 = True
    wp = pack_weight(weight, dtype)
    t_ours = timeit(lambda: depth_layer_forward(feat, weight, bias, wp))
    t_conv = timeit(lambda: F.conv2d(feat, wd, bd)) if only is None else 0.0
    t_conv_widen = timeit(lambda: F.conv2d(feat, wd, bd).float()) if only is None else 0.0
    byts = feat.numel() * feat.element_size() + N * n_out * h * w * 4
    print(f"{dtype}: wgmma {t_ours:.1f} us ({byts / t_ours * 1e-3:.0f} GB/s algorithmic) | cuDNN {t_conv:.1f} us | cuDNN + .float() {t_conv_widen:.1f} us")
