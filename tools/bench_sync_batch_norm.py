"""Time one rank of SyncBatchNorm training: torch's converted nn.SyncBatchNorm against the swapped modules (FusedSyncBatchNorm, and the
SpatialGRU's per-step synced path), eagerly, without CUDA graphs.

    python tools/bench_sync_batch_norm.py [--steps 30] [--out results.json]                         # one GPU
    torchrun --nproc_per_node N tools/bench_sync_batch_norm.py [--steps 30] [--out results.json]    # N GPUs, one rank each

On one GPU the script makes a one-rank NCCL group.  Neither torch's SyncBatchNorm nor FusedSyncBatchNorm synchronizes at world size 1,
so both sides' synced Functions are called directly: torch's ``torch.nn.modules._functions.SyncBatchNorm`` (batch_norm_stats, an
all_gather_into_tensor, batch_norm_gather_stats_with_counts, the elementwise kernels) and ours (local statistics, the gather, the
gathered finalize and apply).  This times the compute plus one collective launch per norm call, not an exchange between GPUs.
Under torchrun with two or more ranks the modules synchronize by themselves and this is the real exchange.

Each case runs --steps times after 3 warm-up runs.  Before every run the ranks meet at a barrier and a 256 MiB buffer is overwritten
so L2 holds none of the case's data.  The run is timed with CUDA events, and each rank prints the median in ms.  The card's name,
power limit and top SM clock are printed first, from the same run.

Cases, per rank, training mode, fp32, forward + backward:
  temporal -- the whole TemporalModel (receptive field 3) at cfg3 = baseline.yml (b 3, s 3, 200 x 200) through temporal_model_forward,
              with the entry, causal-convolution and pyramid-pooling swaps; every norm a converted SyncBatchNorm, against those norms
              swapped by use_fused_sync_batch_norm
  future   -- the 3-GRU FuturePrediction at baseline.yml (b 3, 4 steps of 200 x 200): the reference GRUs with converted norms, against
              use_fused_sync_batch_norm + use_tensor_core_future_prediction (the Bottlenecks' norms stay torch's SyncBatchNorm in both)
  bottleneck -- one Bottleneck at baseline.yml (12 maps = b 3 x 4 steps, 64 channels, 200 x 200): the reference block with converted
              norms, against use_tensor_core_sync_bottlenecks (TensorCoreBottleneck over FusedSyncBatchNorm norms)
  future+bottlenecks -- the future case with use_tensor_core_sync_bottlenecks added to ours: the whole FuturePrediction on the kernels
The first two cases are kept as they were, so their numbers stay comparable across versions.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import socket
import subprocess
import sys

import torch
import torch.distributed as dist
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fiery_b200 import batch_norm as BN  # noqa: E402
from fiery_b200 import bottleneck as BK  # noqa: E402
from fiery_b200 import future_prediction as FP  # noqa: E402
from fiery_b200 import install  # noqa: E402
from fiery_b200.temporal import temporal_model_forward  # noqa: E402
from oracle import future_oracle as FO  # noqa: E402
from oracle import temporal_oracle as TO  # noqa: E402

TEMPORAL = (3, 3, 200, 200)                  # cfg3: b, s, X, Y
FUTURE = (3, 4, 200, 200)                    # b, T, X, Y
HIDDEN, LATENT = 64, 32


def _init():
    """(rank, world, device): torchrun's group, or a one-rank NCCL group"""
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        dist.init_process_group("nccl")
        dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    else:
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("nccl", rank=0, world_size=1)
        dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    return dist.get_rank(), dist.get_world_size(), dev


def _force_sync():
    """At world size 1, make both sides run their synced Functions over the one-rank group."""
    from torch.nn.modules._functions import SyncBatchNorm as TorchSync

    def group_of(norm):
        batch_stats = norm.training or (norm.running_mean is None and norm.running_var is None)
        return (norm.process_group or dist.group.WORLD) if batch_stats and norm.training else None
    BN.sync_group = group_of
    FP.sync_group = group_of
    BK.sync_group = group_of

    def torch_synced(self, x):                  # nn.SyncBatchNorm.forward with need_sync forced
        self._check_input_dim(x)
        factor = 0.0 if self.momentum is None else self.momentum
        if self.training and self.track_running_stats:
            self.num_batches_tracked.add_(1)
            factor = 1.0 / float(self.num_batches_tracked) if self.momentum is None else self.momentum
        return TorchSync.apply(x, self.weight, self.bias, self.running_mean, self.running_var, self.eps, factor,
                               self.process_group or dist.group.WORLD, 1)
    nn.SyncBatchNorm.forward = torch_synced     # FusedSyncBatchNorm has its own forward


def _time(fn, steps):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    times = []
    for _ in range(steps + 3):
        dist.barrier()
        flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times = sorted(times[3:])
    return times[len(times) // 2]


def _step(f, leaves):
    def g():
        y = f()
        y.backward(torch.ones_like(y))
        for t in leaves:
            t.grad = None
    return g


def _temporal_cases(dev):
    b, s, X, Y = TEMPORAL
    torch.manual_seed(0)
    model = TO.TemporalModel(70, 3, (X, Y), start_out_channels=64)
    holder = type("M", (), {"temporal_model": model})()
    install.use_tensor_core_temporal_model(holder)
    install.use_tensor_core_causal_convs(holder)
    install.use_tensor_core_pyramid_pooling(holder)
    ref = nn.SyncBatchNorm.convert_sync_batchnorm(model).to(dev).train()
    ours = copy.deepcopy(ref)
    install.use_fused_sync_batch_norm(type("M", (), {"temporal_model": ours})())
    bev = torch.randn(b, s, 64, X, Y, device=dev, requires_grad=True)
    ego = torch.randn(b, s, 6, device=dev)
    leaves = [bev] + list(ref.parameters()) + list(ours.parameters())
    yield "temporal", _step(lambda: temporal_model_forward(ref, bev, ego), leaves), \
        _step(lambda: temporal_model_forward(ours, bev, ego), leaves)


def _future_cases(dev):
    b, T, X, Y = FUTURE
    torch.manual_seed(7)
    ref = nn.SyncBatchNorm.convert_sync_batchnorm(FO.FuturePrediction(HIDDEN, LATENT)).to(dev).train()
    x = torch.randn(b, 1, LATENT, 1, 1, device=dev, requires_grad=True)
    h0 = torch.randn(b, HIDDEN, X, Y, device=dev, requires_grad=True)
    xin = lambda: x.expand(b, T, LATENT, X, Y)                       # noqa: E731
    for name, bottlenecks in (("future", False), ("future+bottlenecks", True)):
        holder = nn.Module()
        holder.future_prediction = copy.deepcopy(ref)
        install.use_fused_sync_batch_norm(holder)
        install.use_tensor_core_future_prediction(holder)
        if bottlenecks:
            install.use_tensor_core_sync_bottlenecks(holder)
        ours = holder.future_prediction
        leaves = [x, h0] + list(ref.parameters()) + list(ours.parameters())
        yield name, _step(lambda: ref(xin(), h0), leaves), _step(lambda: ours(xin(), h0), leaves)


def _bottleneck_cases(dev):
    b, T, X, Y = FUTURE
    torch.manual_seed(7)
    ref = nn.SyncBatchNorm.convert_sync_batchnorm(FO.Bottleneck(HIDDEN)).to(dev).train()
    holder = nn.Module()
    holder.future_prediction = nn.Module()
    holder.future_prediction.res_blocks = nn.ModuleList([nn.Sequential(copy.deepcopy(ref))])
    install.use_tensor_core_sync_bottlenecks(holder)
    ours = holder.future_prediction.res_blocks[0][0]
    if not isinstance(ours, BK.TensorCoreBottleneck):
        raise SystemExit("the Bottleneck was not swapped")
    x = torch.randn(b * T, HIDDEN, X, Y, device=dev, requires_grad=True)
    leaves = [x] + list(ref.parameters()) + list(ours.parameters())
    yield "bottleneck", _step(lambda: ref(x), leaves), _step(lambda: ours(x), leaves)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these are GPU timings")
    rank, world, dev = _init()
    try:
        info = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
        print(f"# rank {rank}/{world}: {info}", flush=True)
        if world == 1:
            _force_sync()
        rows = []
        for cases in (_temporal_cases, _future_cases, _bottleneck_cases):
            for name, ref, ours in cases(dev):
                t_ref, t_ours = _time(ref, a.steps), _time(ours, a.steps)
                row = dict(rank=rank, world=world, case=name, pass_="fwd+bwd", precision="fp32", torch_sync_ms=round(t_ref, 3),
                           ours_ms=round(t_ours, 3), speedup=round(t_ref / t_ours, 2),
                           note="one-rank group: compute + one collective launch per norm" if world == 1 else "real exchange")
                rows.append(row)
                print(json.dumps(row), flush=True)
            torch.cuda.empty_cache()
        if a.out and rank == 0:
            with open(a.out, "w") as fh:
                json.dump({"gpu": info, "world": world, "rows": rows}, fh, indent=1)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
