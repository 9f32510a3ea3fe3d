"""Time the temporal block's pyramid pooling and aggregation on the kernels against the reference's, by CUDA graph replay.

    python tools/bench_temporal_tail.py [--steps 30] [--out results.json] [--profile DIR]

Each case is captured once in a CUDA graph and replayed; before every replay a 256 MiB buffer is overwritten so L2 holds none of the
case's data, and the replay alone is timed with CUDA events.  The reported figure is the median over --steps replays, in us.  The card's
name, power limit and top SM clock are printed first, from the same run.

Cases (b x s frames of X x Y; fp32, and AMP fp16 via autocast), each as forward only and forward + backward:
  sums        -- spatial_sums of the 64-channel block input as TemporalModel.forward permutes it (forward only), against the HBM bound
                 of reading it once (3.35 TB/s); the row gives the GB/s reached
  aggregation -- the second block's aggregation (3 x 32 path channels + 21 pooled -> 64): the reference's cat of the paths and the
                 broadcast pooled vector + cuDNN Conv3d, against temporal_aggregation (fp32 whatever the autocast)
  block       -- the second TemporalBlock with the entry and causal swaps, without and with the pyramid-pooling swap
  model       -- the whole TemporalModel (receptive field 3, training mode) through temporal_model_forward, entry + causal swaps without
                 and with the pyramid-pooling swap
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
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fiery_b200 import install  # noqa: E402
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


def _swap(m, pool):
    h = type("M", (), {"temporal_model": m})()
    install.use_tensor_core_temporal_model(h)
    install.use_tensor_core_causal_convs(h)
    if pool:
        install.use_tensor_core_pyramid_pooling(h)
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


def _cases(workload, backward):
    b, s, X, Y = WORKLOADS[workload]
    if not backward:
        x = torch.randn(b, s, 64, X, Y, device="cuda").permute(0, 2, 1, 3, 4)
        yield "sums", 4.0 * x.numel(), lambda: x.mean(dim=(3, 4)), lambda: torch.ops.fiery_b200.spatial_sums(x)
    torch.manual_seed(1)
    paths = [torch.randn(b, 32, s, X, Y, device="cuda", requires_grad=backward) for _ in range(3)]
    pooled = torch.randn(b, 21, s, device="cuda", requires_grad=backward)
    weight = (torch.randn(64, 117, 1, 1, 1, device="cuda") / 117 ** 0.5).requires_grad_(backward)
    leaves = paths + [pooled, weight]
    ref = lambda: F.conv3d(torch.cat(paths + [pooled[..., None, None].expand(b, 21, s, X, Y)], 1), weight)
    ours = lambda: torch.ops.fiery_b200.temporal_aggregation(paths, weight, pooled)
    yield "aggregation", None, _run(ref, backward, leaves), _run(ours, backward, leaves)
    entry, both = _models(workload)
    xb = torch.randn(b, 64, s, X, Y, device="cuda", requires_grad=backward)
    yield "block", None, _run(lambda: entry.model[1](xb), backward, [xb]), _run(lambda: both.model[1](xb), backward, [xb])
    bev = torch.randn(b, s, 64, X, Y, device="cuda", requires_grad=backward)
    ego = torch.randn(b, s, 6, device="cuda")
    yield "model", None, _run(lambda: temporal_model_forward(entry, bev, ego), backward, [bev]), \
        _run(lambda: temporal_model_forward(both, bev, ego), backward, [bev])


def _profile(out_dir):
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(out_dir, exist_ok=True)
    b, s, X, Y = WORKLOADS["cfg3"]
    entry, both = _models("cfg3")
    bev = torch.randn(b, s, 64, X, Y, device="cuda", requires_grad=True)
    ego = torch.randn(b, s, 6, device="cuda")
    for tag, m in (("entry_and_causal", entry), ("entry_causal_and_pooling", both)):
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
