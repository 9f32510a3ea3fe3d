"""Time the future prediction's SpatialGRU on the kernels (torch.ops.fiery_b200.spatial_gru) against the reference module, by CUDA
graph replay.

    python tools/bench_spatial_gru.py [--steps 30] [--out results.json] [--profile DIR]

Each case is captured once in a CUDA graph and replayed; before every replay a 256 MiB buffer is overwritten so L2 holds none of the
case's data, and the replay alone is timed with CUDA events.  The reported figure is the median over --steps replays, in us.  The card's
name, power limit and top SM clock are printed first, from the same run.  All cases run in training mode (batch statistics, running
statistics updated once per step).

Cases (fp32, and AMP fp16 via autocast), each as forward only and forward + backward:
  conv_gates_g0 / conv_state_g0 / conv_gates_g1 / conv_state_g1 -- forward only: one step's convolutions of all b x T maps, the
           gates' [x, h] -> [u, r] (2 C_h outputs) and the state's [x, q] -> s, GRU 0 (x 32 channels) and GRU 1 (x 64), on the GRU's
           kernels with plain stores (fiery_conv3x3_forward) against nn.Conv2d over the concatenated input (cuDNN TF32, under AMP
           fp16 as autocast runs it)
  gru0   -- GRU 0: input the latent sample (b, 1, 32, 1, 1) broadcast over the steps and the map, hidden 64 (96 -> 64 channels)
  gru1   -- GRU 1: input a (b, T, 64, X, Y) map, hidden 64 (128 -> 64 channels)
  future -- the whole FuturePrediction (3 GRUs with 3 Bottlenecks each; the Bottlenecks stay torch's in both)
The GRU rows also give the TFLOP/s of the three 3x3 convolutions per step (forward: 2 * pixels * 9 * C_in * (2 C_h + C_h); the
backward counts twice that again) and the time they would take at the data sheet's 495 TFLOP/s (dense TF32, H100 SXM).
Workloads: fp_nusc = baseline.yml (b 3, T 4, 200 x 200), fp_lyft = lyft/baseline.yml (b 3, T 5, 200 x 200).

--profile DIR: a separate torch.profiler run of one forward + backward of GRU 1 at fp_nusc, reference and swapped, writing the per-op
CUDA time tables to DIR.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fiery_b200 import install  # noqa: E402
from fiery_b200.future_prediction import TensorCoreSpatialGRU  # noqa: E402
from oracle import future_oracle as FO  # noqa: E402

WORKLOADS = {"fp_nusc": (3, 4, 200, 200), "fp_lyft": (3, 5, 200, 200)}
PEAK_TF32 = 495e12
HIDDEN, LATENT = 64, 32


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


def _run(f, backward, leaves):
    def g():
        y = f()
        if backward:
            y.float().backward(torch.ones_like(y, dtype=torch.float32))
            for t in leaves:
                t.grad = None
    return g


def _flops(b, T, X, Y, cx, backward):
    f = 2.0 * b * T * X * Y * 9 * (cx + HIDDEN) * 3 * HIDDEN
    return f * (3 if backward else 1)


def _gru_case(workload, index, backward):
    b, T, X, Y = WORKLOADS[workload]
    torch.manual_seed(index)
    cx = LATENT if index == 0 else HIDDEN
    ref = FO.SpatialGRU(cx, HIDDEN).cuda().train()
    ours = TensorCoreSpatialGRU.from_module(copy.deepcopy(ref))
    if index == 0:
        x = torch.randn(b, 1, cx, 1, 1, device="cuda", requires_grad=backward)
        xin = lambda: x.expand(b, T, cx, X, Y)                       # noqa: E731
    else:
        x = torch.randn(b, T, cx, X, Y, device="cuda", requires_grad=backward)
        xin = lambda: x                                              # noqa: E731
    h0 = torch.randn(b, HIDDEN, X, Y, device="cuda", requires_grad=backward)
    leaves = [x, h0] + list(ref.parameters()) + list(ours.parameters())
    return (_flops(b, T, X, Y, cx, backward), _run(lambda: ref(xin(), h0), backward, leaves),
            _run(lambda: ours(xin(), h0), backward, leaves))


def _future_case(workload, backward):
    b, T, X, Y = WORKLOADS[workload]
    torch.manual_seed(7)
    ref = FO.FuturePrediction(HIDDEN, LATENT).cuda().train()
    holder = type("M", (torch.nn.Module,), {})()
    holder.future_prediction = copy.deepcopy(ref)
    install.use_tensor_core_future_prediction(holder)
    ours = holder.future_prediction
    x = torch.randn(b, 1, LATENT, 1, 1, device="cuda", requires_grad=backward)
    h0 = torch.randn(b, HIDDEN, X, Y, device="cuda", requires_grad=backward)
    leaves = [x, h0] + list(ref.parameters()) + list(ours.parameters())
    xin = lambda: x.expand(b, T, LATENT, X, Y)                       # noqa: E731
    return None, _run(lambda: ref(xin(), h0), backward, leaves), _run(lambda: ours(xin(), h0), backward, leaves)


def _conv_case(workload, cx, n_out):
    from fiery_b200.future_prediction import conv3x3_desc, conv3x3_forward, conv3x3_pack
    b, T, X, Y = WORKLOADS[workload]
    maps = b * T
    torch.manual_seed(cx + n_out)
    conv = torch.nn.Conv2d(cx + HIDDEN, n_out, 3, padding=1, bias=False).cuda()
    x0 = torch.randn(maps, cx, X, Y, device="cuda")
    x1 = torch.randn(maps, HIDDEN, X, Y, device="cuda")
    segs = (n_out // 2, n_out // 2) if n_out > HIDDEN else (n_out, 0)
    d = conv3x3_desc(maps, X, Y, (cx, HIDDEN), segs)
    packed = conv3x3_pack(conv.weight, d)
    y0 = torch.empty(maps, segs[0], X, Y, device="cuda")
    y1 = torch.empty(maps, segs[1], X, Y, device="cuda") if segs[1] else None
    flops = 2.0 * maps * X * Y * 9 * (cx + HIDDEN) * n_out
    return flops, lambda: conv(torch.cat([x0, x1], 1)), lambda: conv3x3_forward(d, x0, x1, packed, y0, y1)


def _cases(workload, backward):
    if not backward:
        for cx, tag in ((LATENT, "g0"), (HIDDEN, "g1")):
            yield (f"conv_gates_{tag}",) + _conv_case(workload, cx, 2 * HIDDEN)
            yield (f"conv_state_{tag}",) + _conv_case(workload, cx, HIDDEN)
    yield ("gru0",) + _gru_case(workload, 0, backward)
    yield ("gru1",) + _gru_case(workload, 1, backward)
    yield ("future",) + _future_case(workload, backward)


def _profile(out_dir):
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(out_dir, exist_ok=True)
    _, ref, ours = _gru_case("fp_nusc", 1, True)
    for tag, fn in (("reference", ref), ("swapped", ours)):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=30)
        with open(os.path.join(out_dir, f"profile_gru1_fp_nusc_fwd_bwd_{tag}.txt"), "w") as fh:
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
                for name, flops, ref, ours in _cases(workload, backward):
                    with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                        t_ref = _time(ref, a.steps)
                        t_ours = _time(ours, a.steps)
                    row = dict(workload=workload, case=name, pass_="fwd+bwd" if backward else "fwd", precision="amp" if amp else "fp32",
                               reference_us=round(t_ref, 1), ours_us=round(t_ours, 1), speedup=round(t_ref / t_ours, 2))
                    if flops is not None:
                        row.update(tflops=round(flops / t_ours / 1e6, 1), bound_us=round(flops / PEAK_TF32 * 1e6, 1))
                        if name.startswith("conv"):
                            row.update(reference_tflops=round(flops / t_ref / 1e6, 1))
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
