"""Time the first BEV convolution's backward (fiery_b200/csrc/bev_conv_bwd.cu) against cuDNN's TF32 backward of the same layer.

    python tools/bench_first_conv_backward.py [--steps 50] [--warmup 10]

Workloads: the decoder input of cfg2_static_lss_b8 (8 frames of 200 x 200 x 64) and of cfg4_pon (12 frames of 400 x 200 x 64), both
channel-last fp32.  Every step is captured in a CUDA graph and timed by replay with CUDA events, with a 256 MB L2 flush before each
step (the method of tools/bench_deterministic.py); the median of --steps replays is reported:
  dgrad   the transposed weight pack + the input-gradient kernel
  wgrad   the weight-gradient kernel + the reduce of its chunk partials
  both    all of the above (what FirstConv's backward launches when both gradients are needed and the weight has changed)
  cudnn   aten.convolution_backward under allow_tf32 on the same channels-last tensors with the matching output_mask
  module  FirstConv forward + backward against nn.Conv2d forward + backward (cuDNN TF32), both gradients
Achieved TFLOP/s use the shape-derived count 2 * 49 * 64 * 64 * B * Ho * Wo per gradient (32.1 GFLOP at 8 frames of 200 x 200).
Prints the card, its power limit and max SM clock, one line per workload and a final JSON line.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fiery_b200.bev_conv import (FirstConv, first_conv_backward_data, first_conv_backward_weight,  # noqa: E402
                                 pack_weight_transposed)
from tools.bench_deterministic import card, timed  # noqa: E402

DEV = torch.device("cuda:0")
WORKLOADS = [("cfg2_static_lss_b8", 8, 200, 200), ("cfg4_pon", 12, 400, 200)]


def graphed(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def workload(name, B, H, W, steps, warmup, flush):
    torch.manual_seed(0)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    x = torch.randn(B, H, W, 64, device=DEV).permute(0, 3, 1, 2)
    gy = torch.randn(B, Ho, Wo, 64, device=DEV).permute(0, 3, 1, 2)
    w = torch.randn(64, 64, 7, 7, device=DEV) * 0.02
    ws = torch.empty(18 * 49 * 64 * 64 * 4, dtype=torch.uint8, device=DEV)

    def dgrad():
        first_conv_backward_data(gy, pack_weight_transposed(w), H, W)

    def wgrad():
        first_conv_backward_weight(x, gy, ws)

    def both():
        dgrad()
        wgrad()

    def cudnn(mask):
        return lambda: torch.ops.aten.convolution_backward(gy, x, w, None, [2, 2], [3, 3], [1, 1], False, [0, 0], 1, mask)

    fc = FirstConv().to(DEV)
    conv = nn.Conv2d(64, 64, 7, 2, 3, bias=False).to(DEV).to(memory_format=torch.channels_last)
    with torch.no_grad():
        conv.weight.copy_(fc.weight)
    xg = x.detach().clone().requires_grad_(True)

    def module(m):
        def step():
            xg.grad = None
            m.weight.grad = None
            m(xg).backward(gy)
        return step

    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        t = {k: timed(graphed(f).replay, steps, warmup, flush) for k, f in (
            ("dgrad", dgrad), ("wgrad", wgrad), ("both", both), ("cudnn_dgrad", cudnn([True, False, False])),
            ("cudnn_wgrad", cudnn([False, True, False])), ("cudnn_both", cudnn([True, True, False])),
            ("first_conv_fwd_bwd", module(fc)), ("conv2d_fwd_bwd", module(conv)))}
    finally:
        torch.backends.cudnn.allow_tf32 = old
    flop = 2 * 49 * 64 * 64 * B * Ho * Wo
    tf = {k: (2 if k in ("both", "cudnn_both") else 1) * flop / (v * 1e-3) / 1e12 for k, v in t.items() if "fwd_bwd" not in k}
    return dict(workload=name, frames=B, H=H, W=W, gflop_per_gradient=flop / 1e9, ms=t, tflops=tf)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    a.steps = max(a.steps, 30)
    name, limits = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {limits}", flush=True)
    flush = torch.empty(256 << 18, device=DEV)            # 256 MB
    rows = []
    for wl in WORKLOADS:
        r = workload(*wl, a.steps, a.warmup, flush)
        rows.append(r)
        ms, tf = r["ms"], r["tflops"]
        print(f"{r['workload']:20s} ({r['frames']} x {r['H']} x {r['W']}, {r['gflop_per_gradient']:.1f} GFLOP per gradient)", flush=True)
        for ours, ref in (("dgrad", "cudnn_dgrad"), ("wgrad", "cudnn_wgrad"), ("both", "cudnn_both")):
            print(f"    {ours:6s} {ms[ours] * 1e3:9.1f} us {tf[ours]:6.1f} TFLOP/s   cuDNN TF32 {ms[ref] * 1e3:9.1f} us {tf[ref]:6.1f} TFLOP/s"
                  f"   x{ms[ref] / ms[ours]:.2f}", flush=True)
        print(f"    FirstConv fwd+bwd {ms['first_conv_fwd_bwd'] * 1e3:9.1f} us   nn.Conv2d fwd+bwd {ms['conv2d_fwd_bwd'] * 1e3:9.1f} us"
              f"   x{ms['conv2d_fwd_bwd'] / ms['first_conv_fwd_bwd']:.2f}", flush=True)
    print(json.dumps(dict(card=name, limits=limits, steps=a.steps, results=rows)))


if __name__ == "__main__":
    main()
