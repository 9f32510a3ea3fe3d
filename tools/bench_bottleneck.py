"""Time the future prediction's Bottlenecks on the kernels (torch.ops.fiery_b200.bottleneck) against the reference module, by CUDA
graph replay.

    python tools/bench_bottleneck.py [--steps 30] [--out results.json]

Each case is captured once in a CUDA graph and replayed; before every replay a 256 MiB buffer is overwritten so L2 holds none of the
case's data, and the replay alone is timed with CUDA events.  The reported figure is the median over --steps replays, in us.  The card's
name, power limit and top SM clock are printed first, from the same run.  All cases run in training mode (batch statistics, running
statistics updated once per call).

Cases (fp32, and AMP fp16 via autocast), each as forward only and forward + backward, reference module -> ours:
  bottleneck -- one Bottleneck(64) on the (b T, 64, 200, 200) maps
  stack      -- one res_blocks[i]: three Bottlenecks in a row
  future     -- the whole FuturePrediction with the SpatialGRU swap (reference column) against the SpatialGRU swap plus the
                Bottleneck swap (ours column)
The bottleneck and stack rows also give bound_us: the bytes the fused chain moves at the least (every map it reads or writes, once
per pass that touches it, counted from the shapes below) over the data sheet's 3.35 TB/s (HBM3, H100 SXM), and every row the peak
memory one eager forward + backward allocates (reference, ours).
Workloads: fp_nusc = baseline.yml (b 3, T 4, 200 x 200), fp_lyft = lyft/baseline.yml (b 3, T 5, 200 x 200).
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
from fiery_b200.bottleneck import TensorCoreBottleneck  # noqa: E402
from oracle import future_oracle as FO  # noqa: E402

WORKLOADS = {"fp_nusc": (3, 4, 200, 200), "fp_lyft": (3, 5, 200, 200)}
PEAK_BYTES = 3.35e12
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


def _peak_mib(fn):
    """MiB one eager call of fn allocates at its peak, above what was allocated before it"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def _run(f, backward, leaves):
    def g():
        y = f()
        if backward:
            y.float().backward(torch.ones_like(y, dtype=torch.float32))
            for t in leaves:
                t.grad = None
    return g


def bound_bytes(maps, pixels, c, backward):
    """The fused chain's map traffic in bytes: forward x, y1 (written, read by the statistics and the 3x3), y2 (written, read by
    the statistics and the 1x1), y3 (written, read by the statistics and the apply), x again and out: 6C + 6M floats per pixel;
    backward bn3 (y3 and g twice, dy3), dW_up (y2, dy3), da2 (dy3 -> M), bn2 (5M), dW_conv (y1, dy2), da1 (dy2 -> M), bn1 (5M),
    dW_down (x, dy1), dx (dy1, g, dx): 10C + 18M more."""
    m = c // 2
    floats = 6 * c + 6 * m + ((10 * c + 18 * m) if backward else 0)
    return 4.0 * maps * pixels * floats


def _block_case(workload, n_blocks, backward):
    b, T, X, Y = WORKLOADS[workload]
    torch.manual_seed(n_blocks)
    ref = torch.nn.Sequential(*[FO.Bottleneck(HIDDEN) for _ in range(n_blocks)]).cuda().train()
    ours = torch.nn.Sequential(*[TensorCoreBottleneck.from_module(blk) for blk in copy.deepcopy(ref)])
    x = torch.randn(b * T, HIDDEN, X, Y, device="cuda", requires_grad=backward)
    leaves = [x] + list(ref.parameters()) + list(ours.parameters())
    return (n_blocks * bound_bytes(b * T, X * Y, HIDDEN, backward), _run(lambda: ref(x), backward, leaves),
            _run(lambda: ours(x), backward, leaves))


def _future_case(workload, backward):
    b, T, X, Y = WORKLOADS[workload]
    torch.manual_seed(7)
    fp = FO.FuturePrediction(HIDDEN, LATENT).cuda().train()
    holders = []
    for swap_bottlenecks in (False, True):
        holder = type("M", (torch.nn.Module,), {})()
        holder.future_prediction = copy.deepcopy(fp)
        install.use_tensor_core_future_prediction(holder)
        if swap_bottlenecks:
            install.use_tensor_core_bottlenecks(holder)
        holders.append(holder.future_prediction)
    ref, ours = holders
    x = torch.randn(b, 1, LATENT, 1, 1, device="cuda", requires_grad=backward)
    h0 = torch.randn(b, HIDDEN, X, Y, device="cuda", requires_grad=backward)
    leaves = [x, h0] + list(ref.parameters()) + list(ours.parameters())
    xin = lambda: x.expand(b, T, LATENT, X, Y)                       # noqa: E731
    return None, _run(lambda: ref(xin(), h0), backward, leaves), _run(lambda: ours(xin(), h0), backward, leaves)


def _cases(workload, backward):
    yield ("bottleneck",) + _block_case(workload, 1, backward)
    yield ("stack",) + _block_case(workload, 3, backward)
    yield ("future",) + _future_case(workload, backward)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
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
                        peak = (_peak_mib(ref), _peak_mib(ours)) if backward else None
                    row = dict(workload=workload, case=name, pass_="fwd+bwd" if backward else "fwd", precision="amp" if amp else "fp32",
                               reference_us=round(t_ref, 1), ours_us=round(t_ours, 1), speedup=round(t_ref / t_ours, 2))
                    if nbytes is not None:
                        row.update(bound_us=round(nbytes / PEAK_BYTES * 1e6, 1))
                    if peak is not None:
                        row.update(peak_mib_reference=peak[0], peak_mib_ours=peak[1])
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                    del ref, ours
                    torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
