"""Default vs deterministic forward (torch.use_deterministic_algorithms(True)) of the lift and of VoxelsSumming on one GPU.

    python tools/bench_deterministic.py [--steps 50] [--warmup 5]

Lift workloads: 8 / 9 / 12 frames (cfg2_static_lss_b8, cfg3_baseline, cfg4_pon) with NCHW output, channel-last output and the warped
lift (sequences of 4 frames).  Each is captured in a CUDA graph under each setting of the flag and timed by replay with CUDA events;
a 256 MB buffer is rewritten before every step so no step starts with the previous one's data in L2.  VoxelsSumming: the forward of a
bench-sized input (2.4 M rows x 64 channels in 320 000 voxels, ranks sorted) through the C ABI, timed the same way (its plan
synchronises with the host, so it is not captured).  Prints the card and its power limit, one line per workload with the median step
times, the slowdown factor and the deterministic workspace, and a JSON summary as the last line."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fiery_b200 import _lib  # noqa: E402
from fiery_b200.geometry import _stream_ptr  # noqa: E402
from fiery_b200.lift import LiftSplat  # noqa: E402
from fiery_b200.synthetic import CONFIGS, make_calibration, make_egomotion, make_head  # noqa: E402
from fiery_b200.warp import _device_theta  # noqa: E402

DEV = torch.device("cuda:0")


def card():
    name = torch.cuda.get_device_name(DEV)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def timed(step, steps, warmup, flush):
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        flush.zero_()                                     # evict the previous step's lines from L2
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def graphed(fn, deterministic):
    torch.use_deterministic_algorithms(deterministic)
    try:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g), torch.no_grad():
            out = fn()
    finally:
        torch.use_deterministic_algorithms(False)
    return g, out


def lift_workload(name, variant, steps, warmup, flush):
    cfg = CONFIGS[name]
    K, E = make_calibration(cfg, seed=1)
    hd = torch.from_numpy(make_head(cfg, seed=1)).to(DEV)
    Kd, Ed = torch.from_numpy(K).to(DEV), torch.from_numpy(E).to(DEV)
    lift = LiftSplat.from_config(cfg, output_layout="channels_last" if variant == "nhwc" else "contiguous").to(DEV)
    B = cfg.frames
    warp = None
    if variant == "warped":
        s = 4 if B % 4 == 0 else 3
        flow = torch.from_numpy(make_egomotion(B // s, s, seed=2)).to(DEV)
        warp = _device_theta(flow, (float(cfg.x_bound[1]), float(cfg.y_bound[1])), cumulative=True)
    lib = _lib.load()
    layout = _lib.BEV_NHWC if variant == "nhwc" else _lib.BEV_NCHW
    desc, _ = lift._abi_args(DEV, Kd, Ed, torch.float32, layout)
    nbytes = int(lib.fiery_lift_scratch_bytes(desc))
    scratch = torch.zeros(max(1, nbytes // 4), device=DEV) if nbytes else None
    ws = int(lib.fiery_lift_deterministic_workspace_bytes(desc))
    fn = lambda: lift._launch_forward(hd, Kd, Ed, scratch=scratch, warp=warp)   # noqa: E731
    g0, out0 = graphed(fn, False)
    g1, out1 = graphed(fn, True)
    t0 = timed(g0.replay, steps, warmup, flush)
    t1 = timed(g1.replay, steps, warmup, flush)
    err = float((out0 - out1).abs().max() / out0.abs().max())
    return dict(workload=f"{name}/{variant}", frames=B, default_ms=t0, deterministic_ms=t1, slowdown=t1 / t0, workspace_bytes=ws,
                max_rel_diff=err)


def vs_workload(steps, warmup, flush):
    lib = _lib.load()
    n, C = 2_400_000, 64
    gen = torch.Generator(device=DEV).manual_seed(3)
    ranks = torch.randint(0, 320_000, (n,), generator=gen, device=DEV).sort().values
    x = torch.randn(n, C, generator=gen, device=DEV)
    coords = torch.stack([ranks, ranks, ranks], 1).contiguous()
    seg = torch.empty(n, dtype=torch.int32, device=DEV)
    u = ctypes.c_int64(0)
    _lib.check(lib.fiery_voxels_summing_plan(n, ranks.data_ptr(), seg.data_ptr(), ctypes.byref(u), _stream_ptr(DEV)), "plan")
    U = int(u.value)
    sums = torch.empty(U, C, device=DEV)
    kept = torch.empty(U, 3, dtype=torch.int64, device=DEV)
    ws_bytes = int(lib.fiery_voxels_summing_deterministic_workspace_bytes(n, C))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    args = (n, C, C, x.data_ptr(), coords.data_ptr(), seg.data_ptr(), U, sums.data_ptr(), kept.data_ptr())
    t0 = timed(lambda: _lib.check(lib.fiery_voxels_summing_forward(*args, _stream_ptr(DEV)), "vs"), steps, warmup, flush)
    ref = sums.clone()
    t1 = timed(lambda: _lib.check(lib.fiery_voxels_summing_forward_deterministic(*args, ws.data_ptr(), _stream_ptr(DEV)), "vs det"),
               steps, warmup, flush)
    err = float((ref - sums).abs().max() / ref.abs().max())
    return dict(workload="voxels_summing/2.4M x 64", frames=None, default_ms=t0, deterministic_ms=t1, slowdown=t1 / t0,
                workspace_bytes=ws_bytes, max_rel_diff=err)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has nothing to report without one")
    name, limits = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {limits}", flush=True)
    flush = torch.empty(256 << 18, device=DEV)            # 256 MB
    rows = []
    for cfg in ("cfg2_static_lss_b8", "cfg3_baseline", "cfg4_pon"):
        for variant in ("nchw", "nhwc", "warped"):
            rows.append(lift_workload(cfg, variant, a.steps, a.warmup, flush))
            r = rows[-1]
            print(f"{r['workload']:32s} default {r['default_ms']:8.3f} ms  deterministic {r['deterministic_ms']:8.3f} ms  "
                  f"x{r['slowdown']:.2f}  workspace {r['workspace_bytes'] / 2**20:8.1f} MiB  max rel diff {r['max_rel_diff']:.2e}",
                  flush=True)
    r = vs_workload(a.steps, a.warmup, flush)
    rows.append(r)
    print(f"{r['workload']:32s} default {r['default_ms']:8.3f} ms  deterministic {r['deterministic_ms']:8.3f} ms  "
          f"x{r['slowdown']:.2f}  workspace {r['workspace_bytes'] / 2**20:8.1f} MiB  max rel diff {r['max_rel_diff']:.2e}", flush=True)
    print(json.dumps(dict(card=name, limits=limits, results=rows)))


if __name__ == "__main__":
    main()
