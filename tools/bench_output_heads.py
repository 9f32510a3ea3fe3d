"""Time the decoder's output heads on the kernels (FusedOutputHead: cuDNN's 3x3, then torch.ops.fiery_b200.output_head) against the
reference heads, by CUDA graph replay.

    python tools/bench_output_heads.py [--steps 30] [--out results.json]

Each case is captured once in a CUDA graph and replayed; before every replay a 256 MiB buffer is overwritten so L2 holds none of the
case's data, and the replay alone is timed with CUDA events.  The reported figure is the median over --steps replays, in us.  The card's
name, power limit and top SM clock are printed first, from the same run.  All cases run in training mode (batch statistics, running
statistics updated once per call).

Cases (fp32, and AMP fp16 via autocast), each as forward only and forward + backward, reference -> swapped:
  head    -- the segmentation head on the (maps, 64, 200, 200) map
  heads   -- all four heads (segmentation, offset, center with its sigmoid, future flow) on the same map
  decoder -- the whole Decoder (oracle/decoder_oracle.py) with use_tensor_core_output_heads, on (b, T, 64, 200, 200)
The head and heads rows also give the bytes after the 3x3 the swapped heads move at the least, counted from the shapes (per head:
forward two reads of y; backward two passes over y, each reading y, plus dy written: three maps) and that count over the data sheet's
3.35 TB/s (HBM3, H100 SXM), bound_us; every forward + backward row gives the peak memory one eager call allocates (reference, ours).
Workloads: baseline.yml (b 3, T 5: 15 maps) and lyft/baseline.yml (b 3, T 6: 18 maps), 64 channels, 200 x 200.
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
from fiery_b200.decoder import FusedOutputHead  # noqa: E402
from oracle import decoder_oracle as DO  # noqa: E402

WORKLOADS = {"nusc": (3, 5, 200, 200), "lyft": (3, 6, 200, 200)}
C = 64
PEAK_BYTES = 3.35e12
HEADS = ((2, False), (2, False), (1, True), (2, False))


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
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def _loss(out):
    return sum(t.float().sum() for t in (out.values() if isinstance(out, dict) else [out]) if t is not None)


def _run(f, backward, leaves):
    def g():
        out = f()
        if backward:
            _loss(out).backward()
            for t in leaves:
                t.grad = None
    return g


def bound_bytes(maps, pixels, n_heads, backward):
    """bytes after the 3x3 per the swapped heads' passes: forward y read twice, backward y read twice and dy written (the outputs and
    their gradients, n <= 2 channels each, are left out)"""
    return 4.0 * maps * pixels * C * n_heads * (2 + (3 if backward else 0))


def _heads_case(workload, n_heads, backward):
    b, T, X, Y = WORKLOADS[workload]
    torch.manual_seed(n_heads)
    ref = [DO.output_head(C, n, sig).cuda().train() for n, sig in HEADS[:n_heads]]
    ours = [FusedOutputHead.from_module(copy.deepcopy(h)) for h in ref]
    x = torch.randn(b * T, C, X, Y, device="cuda", requires_grad=backward)
    leaves = [x] + [p for m in ref + ours for p in m.parameters()]
    run = lambda hs: lambda: {str(i): h(x) for i, h in enumerate(hs)}      # noqa: E731
    return bound_bytes(b * T, X * Y, n_heads, backward), _run(run(ref), backward, leaves), _run(run(ours), backward, leaves)


def _decoder_case(workload, backward):
    b, T, X, Y = WORKLOADS[workload]
    torch.manual_seed(7)
    ref = DO.Decoder(C, 2, True).cuda().train()
    holder = type("M", (torch.nn.Module,), {})()
    holder.decoder = copy.deepcopy(ref)
    ours = install.use_tensor_core_output_heads(holder).decoder
    x = torch.randn(b, T, C, X, Y, device="cuda", requires_grad=backward)
    leaves = [x] + list(ref.parameters()) + list(ours.parameters())
    return None, _run(lambda: ref(x), backward, leaves), _run(lambda: ours(x), backward, leaves)


def _cases(workload, backward):
    yield ("head",) + _heads_case(workload, 1, backward)
    yield ("heads",) + _heads_case(workload, 4, backward)
    yield ("decoder",) + _decoder_case(workload, backward)


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
                        row.update(bytes_mb=round(nbytes / 1e6, 1), bound_us=round(nbytes / PEAK_BYTES * 1e6, 1))
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
