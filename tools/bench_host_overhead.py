"""Host time per eager call of the four tensor-core layers, at shapes small enough that the kernels are not what is timed.

    python tools/bench_host_overhead.py [--calls 1000] [--repeats 5]

For each layer -- DepthLayer, FirstConv, the temporal entry (three 1x1x1 convolutions of a TemporalBlock) and a causal (2, 3, 3)
convolution -- the forward alone and the forward + backward (input and weight gradients) are called --calls times in a row with one
synchronize at the end, after a warm-up that makes every weight pack.  The figure is the best of --repeats such windows, in us per
call: the Python, dispatcher and launch work each call adds on the host.  One JSON line per case, the card first.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fiery_b200 import ops  # noqa: E402,F401  (registers the operators)
from fiery_b200.bev_conv import FirstConv  # noqa: E402
from fiery_b200.depth_layer import DepthLayer  # noqa: E402


def _cases(dev):
    """name -> (forward, parameters and inputs whose gradients the backward computes)"""
    depth = DepthLayer(112).to(dev)
    feat = torch.randn(1, 128, 8, 16, device=dev, requires_grad=True)
    first = FirstConv().to(dev)
    bev = torch.randn(1, 64, 16, 16, device=dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    x_entry = torch.randn(1, 64, 2, 8, 8, device=dev, requires_grad=True)
    w_entry = [nn.Parameter(torch.randn(32, 64, 1, 1, 1, device=dev) * 0.1) for _ in range(3)]
    x_causal = torch.randn(1, 32, 2, 8, 8, device=dev, requires_grad=True)
    w_causal = nn.Parameter(torch.randn(32, 32, 2, 3, 3, device=dev) * 0.05)
    return {
        "depth_layer": (lambda: depth(feat), [feat, *depth.parameters()]),
        "first_conv": (lambda: first(bev), [bev, first.weight]),
        "temporal_entry": (lambda: torch.ops.fiery_b200.temporal_entry(x_entry, w_entry, None)[0], [x_entry, *w_entry]),
        "causal_conv3d": (lambda: torch.ops.fiery_b200.causal_conv3d(x_causal, w_causal), [x_causal, w_causal]),
    }


def _us_per_call(fn, calls, repeats):
    best = float("inf")
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t0) / calls * 1e6)
    return best


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_host_overhead.py needs a CUDA device")
    info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": info[0] if info else torch.cuda.get_device_name()}), flush=True)
    dev = torch.device("cuda:0")
    for name, (forward, leaves) in _cases(dev).items():
        def step():
            for t in leaves:
                t.grad = None
            forward().sum().backward()
        for _ in range(3):                                   # makes the packs, loads the kernels
            step()
        print(json.dumps({"layer": name, "forward_us": round(_us_per_call(forward, args.calls, args.repeats), 2),
                          "forward_backward_us": round(_us_per_call(step, args.calls, args.repeats), 2)}), flush=True)


if __name__ == "__main__":
    main()
