"""Time the temporal block's fused 1x1x1 entry against the reference's ops it replaces, by CUDA graph replay.

    python tools/bench_temporal_entry.py [--steps 30] [--out results.json]

Each case is captured once in a CUDA graph and replayed; before every replay a 256 MiB buffer is overwritten so L2 holds none of the
case's data, and the replay alone is timed with CUDA events.  The reported figure is the median over --steps replays, in us.

Cases (b x s frames of X x Y; fp32, and AMP fp16 via autocast):
  block1 -- the first TemporalBlock's entry.  reference: the egopose concat (fiery.py:148-155), TemporalModel's permute, and the four
            Conv3d 70 -> 35, 35, 35, 64 (under AMP with autocast's casts).  fused: temporal_entry on the 64-channel BEV with the
            egopose folded in as a bias.
  block2 -- the second block's entry: three Conv3d 64 -> 32 against temporal_entry on the contiguous (b, 64, s, X, Y) input.
  model  -- the whole TemporalModel (receptive field 3): concat + the reference model (oracle/temporal_oracle.py, the same modules)
            against temporal_model_forward on the swapped model.
each as forward only and forward + backward (input and weight gradients; BatchNorm in train mode).
Workloads: cfg3 = baseline.yml (b 3, s 3, 200 x 200), cfg4 = pon_setting.yml (b 4, s 3, 400 x 200).
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
from fiery_b200.temporal import temporal_model_forward  # noqa: E402
from oracle import temporal_oracle as TO  # noqa: E402

WORKLOADS = {"cfg3": (3, 3, 200, 200), "cfg4": (4, 3, 400, 200)}


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


def _egopose_concat_permuted(bev, ego):
    return TO.egopose_concat(bev, ego).permute(0, 2, 1, 3, 4)


def _cases(workload, backward):
    b, s, X, Y = WORKLOADS[workload]
    torch.manual_seed(0)
    model = TO.TemporalModel(70, 3, (X, Y), start_out_channels=64).cuda().train()
    swapped = copy.deepcopy(model)
    install.use_tensor_core_temporal_model(type("M", (), {"temporal_model": swapped})())
    bev = torch.randn(b, s, 64, X, Y, device="cuda", requires_grad=backward)
    ego = torch.randn(b, s, 6, device="cuda")
    x2 = torch.randn(b, 64, s, X, Y, device="cuda", requires_grad=backward)
    blk1, blk2 = model.model[0], model.model[1]
    c1 = [blk1.convolution_paths[0][0].conv, blk1.convolution_paths[1][0].conv, blk1.convolution_paths[2].conv, blk1.projection[0]]
    c2 = [blk2.convolution_paths[0][0].conv, blk2.convolution_paths[1][0].conv, blk2.convolution_paths[2].conv]
    extra = torch.cat([torch.zeros_like(ego[:, :1]), ego[:, :s - 1]], 1)

    def run(outs_fn):
        def f():
            outs = outs_fn()
            if backward:
                torch.autograd.backward([o.float() for o in outs], [torch.ones_like(o, dtype=torch.float32) for o in outs])
        return f

    def block1_reference():
        xc = _egopose_concat_permuted(bev, ego)        # built once and read by the four convolutions, as in fiery.py:155
        return [c(xc) for c in c1]

    yield "block1", run(block1_reference), \
        run(lambda: torch.ops.fiery_b200.temporal_entry(bev.permute(0, 2, 1, 3, 4), [c.weight for c in c1], extra))
    yield "block2", run(lambda: [c(x2) for c in c2]), run(lambda: torch.ops.fiery_b200.temporal_entry(x2, [c.weight for c in c2], None))
    yield "model", run(lambda: [model(TO.egopose_concat(bev, ego))]), run(lambda: [temporal_model_forward(swapped, bev, ego)])


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
                for name, ref, fused in _cases(workload, backward):
                    with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                        t_ref = _time(ref, a.steps)
                        t_fused = _time(fused, a.steps)
                    row = dict(workload=workload, case=name, pass_="fwd+bwd" if backward else "fwd", precision="amp" if amp else "fp32",
                               reference_us=round(t_ref, 1), fused_us=round(t_fused, 1), speedup=round(t_ref / t_fused, 2))
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as fh:
            json.dump({"gpu": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
