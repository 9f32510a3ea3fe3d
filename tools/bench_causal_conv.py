"""Time the temporal model's causal convolutions on the tensor cores against the reference's pad + Conv3d, by CUDA graph replay.

    python tools/bench_causal_conv.py [--steps 30] [--out results.json] [--profile DIR]

Each case is captured once in a CUDA graph and replayed; before every replay a 256 MiB buffer is overwritten so L2 holds none of the
case's data, and the replay alone is timed with CUDA events.  The reported figure is the median over --steps replays, in us.  The card's
name, power limit and top SM clock are printed first, from the same run.

Cases (b x s frames of X x Y; fp32, and AMP fp16 via autocast), each as forward only and forward + backward (input and weight
gradients):
  b1_k2 / b1_k1 -- the first block's (2,3,3) and (1,3,3) causal convolutions, 35 -> 35 channels
  b2_k2 / b2_k1 -- the second block's, 32 -> 32 channels
                   reference: ConstantPad3d + Conv3d (cuDNN; under AMP in fp16 as autocast runs it); ours: causal_conv3d (fp32)
  model         -- the whole TemporalModel (receptive field 3) through temporal_model_forward, training mode: the temporal-entry swap
                   alone against the entry + causal-convolution swaps.
For the fp32 convolution cases the row also gives our achieved TFLOP/s (2 * C_in * C_out * 9 kt multiply-adds per output pixel-frame
per pass) and GB/s (the tensors each pass must read and write once), and the lower bound each implies on the card's data-sheet rates
(495 TFLOP/s TF32 dense, 3.35 TB/s HBM3), saying which is the larger.
Workloads: cfg3 = baseline.yml (b 3, s 3, 200 x 200), cfg4 = pon_setting.yml (b 4, s 3, 400 x 200).

--profile DIR: a separate torch.profiler run of one forward + backward of the model with each swap, writing the per-op CUDA time table
(entry-only and entry + causal) to DIR.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fiery_b200 import install  # noqa: E402
from fiery_b200.temporal import temporal_model_forward  # noqa: E402
from oracle import temporal_oracle as TO  # noqa: E402

WORKLOADS = {"cfg3": (3, 3, 200, 200), "cfg4": (4, 3, 400, 200)}
CONVS = {"b1_k2": (35, 2), "b1_k1": (35, 1), "b2_k2": (32, 2), "b2_k1": (32, 1)}
PEAK_TF32, PEAK_BW = 495e12, 3.35e12


def _time(fn, steps):
    """median us of a graph replay of fn, L2 flushed before each replay"""
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    times = []
    for _ in range(steps + 3):
        flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3)
    times = sorted(times[3:])
    return times[len(times) // 2]


def _conv_work(workload, c, kt, backward):
    """(flops, bytes) the fp32 pass needs: forward 1 GEMM, backward 2 more; bytes: x and y once each (forward), plus grad_y read twice,
    x read once and grad_x written once (backward); weights are negligible"""
    b, s, X, Y = WORKLOADS[workload]
    n = b * s * X * Y
    flops = 2.0 * c * c * 9 * kt * n * (3 if backward else 1)
    tensor = 4.0 * c * n
    return flops, tensor * (2 + (4 if backward else 0))


def _models(workload):
    b, s, X, Y = WORKLOADS[workload]
    torch.manual_seed(0)
    model = TO.TemporalModel(70, 3, (X, Y), start_out_channels=64).cuda().train()
    entry = copy.deepcopy(model)
    holder = type("M", (), {"temporal_model": entry})()
    install.use_tensor_core_temporal_model(holder)
    both = copy.deepcopy(entry)
    install.use_tensor_core_causal_convs(type("M", (), {"temporal_model": both})())
    return entry, both


def _cases(workload, backward):
    b, s, X, Y = WORKLOADS[workload]
    for name, (c, kt) in CONVS.items():
        torch.manual_seed(1)
        pad = nn.ConstantPad3d((1, 1, 1, 1, kt - 1, 0), 0.0)
        conv = nn.Conv3d(c, c, (kt, 3, 3), bias=False).cuda()
        x = torch.randn(b, c, s, X, Y, device="cuda", requires_grad=backward)

        def run(f):
            def g():
                y = f()
                if backward:
                    y.float().backward(torch.ones_like(y, dtype=torch.float32))
            return g
        yield name, (c, kt), run(lambda: conv(pad(x))), run(lambda: torch.ops.fiery_b200.causal_conv3d(x, conv.weight))
    entry, both = _models(workload)
    bev = torch.randn(b, s, 64, X, Y, device="cuda", requires_grad=backward)
    ego = torch.randn(b, s, 6, device="cuda")

    def model_run(m):
        def g():
            y = temporal_model_forward(m, bev, ego)
            if backward:
                y.float().backward(torch.ones_like(y, dtype=torch.float32))
        return g
    yield "model", None, model_run(entry), model_run(both)


def _profile(out_dir):
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(out_dir, exist_ok=True)
    b, s, X, Y = WORKLOADS["cfg3"]
    entry, both = _models("cfg3")
    bev = torch.randn(b, s, 64, X, Y, device="cuda", requires_grad=True)
    ego = torch.randn(b, s, 6, device="cuda")
    for tag, m in (("entry_only", entry), ("entry_and_causal", both)):
        for _ in range(3):
            temporal_model_forward(m, bev, ego).sum().backward()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            temporal_model_forward(m, bev, ego).sum().backward()
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=40)
        with open(os.path.join(out_dir, f"profile_cfg3_fwd_bwd_{tag}.txt"), "w") as fh:
            fh.write(table)
        print(f"# profile {tag}\n{table}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these are GPU timings")
    info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"# {info}", flush=True)
    rows = []
    for workload in WORKLOADS:
        for backward in (False, True):
            for amp in (False, True):
                for name, shape, ref, ours in _cases(workload, backward):
                    with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                        t_ref = _time(ref, a.steps)
                        t_ours = _time(ours, a.steps)
                    row = dict(workload=workload, case=name, pass_="fwd+bwd" if backward else "fwd", precision="amp" if amp else "fp32",
                               reference_us=round(t_ref, 1), ours_us=round(t_ours, 1), speedup=round(t_ref / t_ours, 2))
                    if shape is not None and not amp:
                        flops, nbytes = _conv_work(workload, *shape, backward)
                        row.update(tflops=round(flops / t_ours / 1e6, 1), gbs=round(nbytes / t_ours / 1e3, 1),
                                   bound_us=round(max(flops / PEAK_TF32, nbytes / PEAK_BW) * 1e6, 1),
                                   bound="tf32" if flops / PEAK_TF32 > nbytes / PEAK_BW else "hbm")
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)
    if a.profile:
        _profile(a.profile)


if __name__ == "__main__":
    main()
