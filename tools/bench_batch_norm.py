"""Time the temporal model's BatchNorm3d (+ ReLU, + skip add) on the fused kernels against torch's, by CUDA graph replay.

    python tools/bench_batch_norm.py [--steps 30] [--out results.json] [--profile DIR]

Each case is captured once in a CUDA graph and replayed; before every replay a 256 MiB buffer is overwritten so L2 holds none of the
case's data, and the replay alone is timed with CUDA events.  The reported figure is the median over --steps replays, in us.  The card's
name, power limit and top SM clock are printed first, from the same run.  All cases run in training mode (batch statistics, running
statistics updated).

Cases (b x s frames of X x Y; fp32, and AMP fp16 via autocast), each as forward only and forward + backward:
  bn_relu_35    -- BatchNorm3d + ReLU of block 1's 35-channel paths: nn.BatchNorm3d + nn.ReLU(inplace=True) against
                   FusedBatchNorm3d.forward_act(relu=True)
  bn_relu_32    -- the same for block 2's 32-channel paths
  bn_relu_add_64 -- the aggregation's 64-channel BatchNorm3d + ReLU + the block's skip add
  block         -- the second TemporalBlock with the entry, causal and pyramid-pooling swaps, without and with the batch-norm swap
  model         -- the whole TemporalModel (receptive field 3) through temporal_model_forward, the same two swap sets
The single-norm rows also give the GB/s the fused kernels reach and the HBM bound at 3.35 TB/s of the bytes they must move: a training
forward reads x twice (statistics, apply) and writes y, plus the residual read; the backward reads x and dy twice (sums, apply) and
writes dx (the residual's gradient is dy itself).
Workloads: cfg3 = baseline.yml (b 3, s 3, 200 x 200), cfg4 = pon_setting.yml (b 4, s 3, 400 x 200).

--profile DIR: a separate torch.profiler run of one forward + backward of the model at cfg3 with each swap set, writing the per-op CUDA
time table to DIR.
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
from fiery_b200.batch_norm import FusedBatchNorm3d  # noqa: E402
from fiery_b200.temporal import temporal_model_forward  # noqa: E402
from oracle import temporal_oracle as TO  # noqa: E402

WORKLOADS = {"cfg3": (3, 3, 200, 200), "cfg4": (4, 3, 400, 200)}
PEAK_BW = 3.35e12


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


def _holder(m):
    return type("M", (), {"temporal_model": m})()


def _swap(m, bn):
    h = _holder(m)
    install.use_tensor_core_temporal_model(h)
    install.use_tensor_core_causal_convs(h)
    install.use_tensor_core_pyramid_pooling(h)
    if bn:
        install.use_fused_batch_norm(h)
    return m


def _models(workload):
    _, _, X, Y = WORKLOADS[workload]
    torch.manual_seed(0)
    model = TO.TemporalModel(70, 3, (X, Y), start_out_channels=64).cuda().train()
    return _swap(copy.deepcopy(model), False), _swap(copy.deepcopy(model), True)


def _run(f, backward, leaves):
    def g():
        y = f()
        if backward:
            y.float().backward(torch.ones_like(y, dtype=torch.float32))
            for t in leaves:
                t.grad = None
    return g


def _norm_case(b, c, s, X, Y, backward, residual):
    torch.manual_seed(c)
    x = torch.randn(b, c, s, X, Y, device="cuda", requires_grad=backward)
    r = torch.randn(b, c, s, X, Y, device="cuda", requires_grad=backward) if residual else None
    bn = nn.BatchNorm3d(c).cuda().train()
    relu = nn.ReLU(inplace=True)
    fused = FusedBatchNorm3d(copy.deepcopy(bn))
    leaves = [x] + ([r] if residual else []) + [bn.weight, bn.bias, fused.weight, fused.bias]
    ref = (lambda: r + relu(bn(x))) if residual else (lambda: relu(bn(x)))
    ours = lambda: fused.forward_act(x, True, r)                          # noqa: E731
    passes = (4 if residual else 3) + (5 if backward else 0)
    return passes * 4.0 * x.numel(), _run(ref, backward, leaves), _run(ours, backward, leaves)


def _cases(workload, backward):
    b, s, X, Y = WORKLOADS[workload]
    yield ("bn_relu_35",) + _norm_case(b, 35, s, X, Y, backward, False)
    yield ("bn_relu_32",) + _norm_case(b, 32, s, X, Y, backward, False)
    yield ("bn_relu_add_64",) + _norm_case(b, 64, s, X, Y, backward, True)
    unfused, fused = _models(workload)
    xb = torch.randn(b, 64, s, X, Y, device="cuda", requires_grad=backward)
    yield "block", None, _run(lambda: unfused.model[1](xb), backward, [xb]), _run(lambda: fused.model[1](xb), backward, [xb])
    bev = torch.randn(b, s, 64, X, Y, device="cuda", requires_grad=backward)
    ego = torch.randn(b, s, 6, device="cuda")
    yield "model", None, _run(lambda: temporal_model_forward(unfused, bev, ego), backward, [bev]), \
        _run(lambda: temporal_model_forward(fused, bev, ego), backward, [bev])


def _profile(out_dir):
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(out_dir, exist_ok=True)
    b, s, X, Y = WORKLOADS["cfg3"]
    unfused, fused = _models("cfg3")
    bev = torch.randn(b, s, 64, X, Y, device="cuda", requires_grad=True)
    ego = torch.randn(b, s, 6, device="cuda")
    for tag, m in (("three_swaps", unfused), ("three_swaps_and_batch_norm", fused)):
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
                for name, nbytes, ref, ours in _cases(workload, backward):
                    with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                        t_ref = _time(ref, a.steps)
                        t_ours = _time(ours, a.steps)
                    row = dict(workload=workload, case=name, pass_="fwd+bwd" if backward else "fwd", precision="amp" if amp else "fp32",
                               reference_us=round(t_ref, 1), ours_us=round(t_ours, 1), speedup=round(t_ref / t_ours, 2))
                    if nbytes is not None:
                        row.update(gbs=round(nbytes / t_ours / 1e3, 1), bound_us=round(nbytes / PEAK_BW * 1e6, 1))
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
